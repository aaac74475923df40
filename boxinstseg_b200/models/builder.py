"""The registry surface (drop-in boundary, SURVEY.md section 8b).

The reference builds heads and losses from config dicts through mmcv registries
(mmdet/models/builder.py:7-59: ``HEADS = LOSSES = MODELS``).  When the reference's ``mmdet`` is
importable the classes of this package are registered INTO its registries with ``force=True``
under the reference's own names, so ``configs/boxinst/*.py`` etc. build the CUDA implementations
unchanged after ``import boxinstseg_b200.models``.  Without mmcv/mmdet (this image) a minimal
registry with the same ``register_module`` / ``build`` behaviour is used.
"""
import inspect

try:                                            # pragma: no cover - mmdet is absent in this image
    from mmdet.models.builder import HEADS, LOSSES
    from mmdet.core.bbox.match_costs.builder import MATCH_COST
    HAVE_MMDET = True
except Exception:                               # noqa: BLE001
    HAVE_MMDET = False

    class Registry:
        """register_module()/build() subset of mmcv.utils.Registry."""

        def __init__(self, name):
            self.name = name
            self.module_dict = {}

        def get(self, key):
            return self.module_dict.get(key)

        def register_module(self, name=None, force=False, module=None):
            def _register(cls):
                key = name or cls.__name__
                if key in self.module_dict and not force:
                    raise KeyError(f'{key} is already registered in {self.name}')
                self.module_dict[key] = cls
                return cls
            return _register(module) if module is not None else _register

        def build(self, cfg, default_args=None):
            if not isinstance(cfg, dict) or 'type' not in cfg:
                raise TypeError(f'cfg must be a dict with a "type" key, got {cfg!r}')
            args = dict(cfg)
            if default_args:
                for k, v in default_args.items():
                    args.setdefault(k, v)
            kind = args.pop('type')
            cls = self.get(kind) if isinstance(kind, str) else kind
            if cls is None:
                raise KeyError(f'{kind} is not in the {self.name} registry')
            if not (inspect.isclass(cls) or callable(cls)):
                raise TypeError(f'type must be a str or class, got {type(cls)}')
            return cls(**args)

    MODELS = Registry('models')
    HEADS = LOSSES = MODELS                      # builder.py:9-15 -- one shared registry
    MATCH_COST = Registry('Match Cost')
    PIPELINES = Registry('pipeline')             # mmdet/datasets/builder.py; filled by `import boxinstseg_b200.datasets`


def register(registry, partial=False, **kw):
    """register_module under the reference's own name.

    Complete replacements (losses, match costs) simply override a same-named reference class.  ``partial=True``
    marks classes that implement only the mask-loss hot path of a reference head: when the reference's class is
    already registered under that name (mmdet importable) the registered class becomes a subclass of BOTH -- this
    package's methods first in the MRO, the reference's own ``__init__`` and every method this package does not
    provide (``training_sample``, ``simple_test``, ``get_masks``, target builders, ...) inherited unchanged -- so
    ``detectors/condinst.py:54-90`` keeps working after ``import boxinstseg_b200.models``."""
    def _do(cls):
        key = kw.get('name') or cls.__name__
        ref = registry.get(key) if partial else None
        if ref is not None and ref is not cls and not issubclass(ref, cls):
            def _init(self, *a, **k):
                ref.__init__(self, *a, **k)                    # every attribute the inherited reference methods use
                post = getattr(cls, '_bxs_post_init', None)
                if post is not None:
                    post(self)
            cls = type(cls.__name__, (cls, ref), {'__init__': _init, '__module__': cls.__module__,
                                                   '__doc__': cls.__doc__, '_bxs_reference_class': ref})
        return registry.register_module(force=True, module=cls, **kw)
    return _do


def build_head(cfg):
    return HEADS.build(cfg)


def build_loss(cfg):
    return LOSSES.build(cfg)
