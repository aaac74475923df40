from .condinst import LogVars, mask_branch_step, parse_losses  # noqa: F401
from .discobox import DiscoBoxSOLOv2, forward_train, momentum_update  # noqa: F401  (registers the class)
from .solo import BoxLevelSet, format_results  # noqa: F401  (registers the class)
