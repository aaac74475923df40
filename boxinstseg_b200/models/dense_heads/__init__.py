from .box2mask_infer import MaskFormerFusionHead  # noqa: F401
from .condinst_mask_head import CondInstMaskHead  # noqa: F401
from .mask_loss_heads import Box2MaskHead, BoxSOLOv2Head, DiscoBoxSOLOv2Head  # noqa: F401
from .meanfield import MeanField  # noqa: F401
from .condinst_box_head import CondInstBoxHead, fcos_get_targets  # noqa: F401
from .condinst_segm_head import CondInstSegmHead  # noqa: F401
