from .condinst import LogVars, mask_branch_step, parse_losses  # noqa: F401
from .solo import BoxLevelSet, DiscoBoxSOLOv2, format_results  # noqa: F401  (registers the classes)
