from .assigner import AssignResult, ClassificationCost, MaskHungarianAssigner  # noqa: F401
from .box_masks import BoxMasks  # noqa: F401
from .mask import encode_mask_results  # noqa: F401
from .match_cost import BoxMatchingCost, projection_profiles  # noqa: F401
