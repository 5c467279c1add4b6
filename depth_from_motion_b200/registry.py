"""Registry / config plumbing at the reference's plugin boundary.

The reference builds its modules from config dicts through mmcv registries
(mmdet3d/models/builder.py:16-96; ``DfMBackbone`` and ``DepthHead`` register into
mmdet's ``BACKBONES`` / ``HEADS``, dfm_backbone.py:11-14, depth_head.py:10-13;
``DfMNeck`` / ``OutdoorImVoxelNeck`` into mmdet3d's ``NECKS``, dfm_neck.py:6-10).

When mmcv/mmdet are importable, ``register_into_mmdet()`` registers the
H100-native classes under the same names with ``force=True`` so an unmodified
``configs/dfm/*.py`` builds them.  mmcv is not installed in this image, so the
module also carries a minimal ``Registry`` + ``Config`` with the same call
shapes (``register_module()``, ``build(cfg)``, ``Config.fromfile``) -- enough to
parse the reference's flat python configs and build the hot-path modules by
``type``.
"""
import copy
import os


class Registry:
    """mmcv.utils.Registry call-compatible subset."""

    def __init__(self, name):
        self.name = name
        self._module_dict = {}

    @property
    def module_dict(self):
        return self._module_dict

    def get(self, key):
        return self._module_dict.get(key)

    def __contains__(self, key):
        return key in self._module_dict

    def register_module(self, name=None, force=False, module=None):
        def _register(cls):
            key = name or cls.__name__
            if key in self._module_dict and not force:
                raise KeyError(f'{key} is already registered in {self.name}')
            self._module_dict[key] = cls
            return cls

        if module is not None:
            return _register(module)
        return _register

    def build(self, cfg, default_args=None):
        if not isinstance(cfg, dict) or 'type' not in cfg:
            raise TypeError('cfg must be a dict with the key "type"')
        args = copy.deepcopy(dict(cfg))
        if default_args:
            for k, v in default_args.items():
                args.setdefault(k, v)
        obj_type = args.pop('type')
        cls = self.get(obj_type) if isinstance(obj_type, str) else obj_type
        if cls is None:
            raise KeyError(f'{obj_type} is not in the {self.name} registry')
        return cls(**args)


BACKBONES = Registry('backbone')
NECKS = Registry('neck')
HEADS = Registry('head')
DETECTORS = Registry('detector')


def build_backbone(cfg):
    """mmdet3d/models/builder.py:31-36."""
    return BACKBONES.build(cfg)


def build_neck(cfg):
    """mmdet3d/models/builder.py:39-44."""
    return NECKS.build(cfg)


def build_head(cfg):
    """mmdet3d/models/builder.py:63-68."""
    return HEADS.build(cfg)


def build_detector(cfg, train_cfg=None, test_cfg=None):
    """mmdet3d/models/builder.py:79-96: ``DfM`` / ``MultiViewDfM`` from a config's ``model``
    dict; ``train_cfg`` / ``test_cfg`` given here must not also be in ``cfg``."""
    assert cfg.get('train_cfg') is None or train_cfg is None, \
        'train_cfg specified in both outer field and model field '
    assert cfg.get('test_cfg') is None or test_cfg is None, \
        'test_cfg specified in both outer field and model field '
    default_args = {k: v for k, v in (('train_cfg', train_cfg), ('test_cfg', test_cfg))
                    if v is not None}
    return DETECTORS.build(cfg, default_args=default_args)


class ConfigDict(dict):
    """Attribute access on nested dicts (mmcv.Config behaviour used by tools)."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return ConfigDict(v) if isinstance(v, dict) and not isinstance(v, ConfigDict) else v


class Config:
    """``mmcv.Config.fromfile`` for flat python configs (no ``_base_``), which is
    what every ``configs/dfm/*.py`` is (SURVEY.md section 5)."""

    def __init__(self, cfg_dict, filename=None):
        self._cfg_dict = ConfigDict(cfg_dict)
        self.filename = filename

    @staticmethod
    def fromfile(filename):
        filename = os.path.abspath(filename)
        scope = {'__file__': filename}
        with open(filename) as f:
            exec(compile(f.read(), filename, 'exec'), scope)
        if '_base_' in scope:
            raise NotImplementedError('_base_ inheritance needs mmcv')
        cfg = {k: v for k, v in scope.items()
               if not k.startswith('__') and not callable(v)
               and type(v).__name__ != 'module'}
        return Config(cfg, filename)

    def __getattr__(self, k):
        return getattr(self._cfg_dict, k)

    def __getitem__(self, k):
        return self._cfg_dict[k]

    def __contains__(self, k):
        return k in self._cfg_dict


def register_into_mmdet():
    """Registers the H100-native classes into the real mmdet / mmdet3d registries
    (same names as the reference, ``force=True``).  Returns False when mmcv/mmdet
    are not installed."""
    try:
        from mmdet.models.builder import BACKBONES as MM_BACKBONES
        from mmdet.models.builder import HEADS as MM_HEADS
    except Exception:  # mmdet absent in this image
        return False
    from . import modules
    MM_BACKBONES.register_module(name='DfMBackbone', force=True,
                                 module=modules.DfMBackbone)
    MM_HEADS.register_module(name='DepthHead', force=True,
                             module=modules.DepthHead)
    # (the detectors DfM / MultiViewDfM are registered locally only: mmdet3d's own stay in
    # place.  LIGAAnchor3DHead and Anchor3DHead are NOT forced into mmdet's registry: the mirrors
    # have forward, get_bboxes and loss, but no backward through their convs, which the
    # detector's forward_train needs;
    # BEVHourglass's forward is the whole module)
    MM_BACKBONES.register_module(name='BEVHourglassB200', force=True,
                                 module=modules.BEVHourglass)
    try:
        from mmdet3d.models.builder import NECKS as MM3D_NECKS
        MM3D_NECKS.register_module(name='DfMNeck', force=True,
                                   module=modules.DfMNeck)
        MM3D_NECKS.register_module(name='OutdoorImVoxelNeck', force=True,
                                   module=modules.OutdoorImVoxelNeck)
    except Exception:
        pass
    try:  # FrustumToVoxel registers into mmdet's NECKS (feature_transformation.py:9-12)
        from mmdet.models.builder import NECKS as MM_NECKS
        MM_NECKS.register_module(name='FrustumToVoxel', force=True,
                                 module=modules.FrustumToVoxel)
    except Exception:
        pass
    return True
