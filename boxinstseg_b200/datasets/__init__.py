"""The data-pipeline side of box supervision: ``GenerateBoxMask`` building ``core.BoxMasks`` rectangles instead of
``BitmapMasks`` arrays.

Importing this package registers it into the pipeline registry under the reference's own name, with ``force=True``:
mmdet's ``PIPELINES`` when mmdet is importable, else ``models.builder.PIPELINES``.  It is an opt-in of its own (a
``custom_imports`` entry next to ``boxinstseg_b200.models``); ``import boxinstseg_b200.models`` alone leaves the
reference's ``GenerateBoxMask`` in place."""
from ..models.builder import HAVE_MMDET
from .pipelines import GenerateBoxMask

if HAVE_MMDET:                                  # pragma: no cover - mmdet is absent in this image
    from mmdet.datasets.builder import PIPELINES
else:
    from ..models.builder import PIPELINES

PIPELINES.register_module(force=True, module=GenerateBoxMask)

__all__ = ['GenerateBoxMask', 'PIPELINES']
