"""Checkpoint key plumbing for the hot-path modules (SURVEY.md section 8(f) row 4).

A reference DfM detector checkpoint stores the hot-path parameters under the
sub-module names of ``mmdet3d/models/detectors/dfm.py:54-76``:

    backbone_stereo.*          -> DfMBackbone
    feature_transformation.*   -> FrustumToVoxel
    neck_3d.*                  -> DfMNeck / OutdoorImVoxelNeck (multiview_dfm.py)
    bbox_head_3d.*             -> Anchor3DHead (MultiViewDfM; mmdet3d-style keys only)
    neck.*                     -> SPPUNetNeck (DfM's image neck, detectors/dfm.py:44) or
                                  FPN (MultiViewDfM's image neck)
    backbone.*                 -> LIGAResNet (DfM's image backbone, detectors/dfm.py:43) or
                                  ResNet (MultiViewDfM's ResNet-101 + DCNv2 image backbone)

and the original LIGA-DfM release uses older names that the reference's
``tools/model_converters/convert_dfm_checkpoints.py:34-63`` renames (first matching
prefix wins, ``:77-81``).  The subset of that table that decides where hot-path
parameters end up is restated here so a LIGA-style ``model_state`` can be read
directly; all other prefixes (``neck_2d``, the heads' decoding) are left untouched because
those modules stay PyTorch on the caller's side.
"""
from collections import OrderedDict

# (old substring, new substring), in the reference's matching order
# (convert_dfm_checkpoints.py:49-63, without the lidar teacher's rows).  The first five rows
# cover the keys that contain 'backbone_3d'; they are all ``load_hot_path`` applies.
_LIGA_RENAMES = (
    ('backbone_3d.feature_backbone', 'backbone'),
    ('backbone_3d.feature_neck', 'neck'),
    ('backbone_3d.sem_neck', 'neck_2d'),
    ('backbone_3d.rpn3d_convs', 'feature_transformation.voxel_convs'),
    ('backbone_3d', 'backbone_stereo'),
    ('backbone_2d.rpn3d_conv2', 'backbone_3d.compress_conv'),
    ('backbone_2d.rpn3d_conv3', 'backbone_3d.bev_hourglass'),
    ('dense_head_2d.bbox_head', 'bbox_head_2d'),
    ('dense_head.rpn3d_cls_convs', 'bbox_head_3d.cls_convs'),
    ('dense_head.rpn3d_bbox_convs', 'bbox_head_3d.reg_convs'),
    ('dense_head.conv_cls', 'bbox_head_3d.conv_cls'),
    ('dense_head.conv_box', 'bbox_head_3d.conv_reg'),
    ('dense_head.conv_dir_cls', 'bbox_head_3d.conv_dir_cls'),
    ('dense_head.norm_imitation', 'norm_imitation'),
    ('dense_head.conv_imitation', 'conv_imitation'),
)
_LIGA_HOT_PATH_RENAMES = _LIGA_RENAMES[:5]

# detector entries that only training builds (the LiDAR teacher, the 2-D head and neck, the
# imitation layers): load_detector skips and reports them
TRAINING_ONLY_PREFIXES = ('lidar_model.', 'neck_2d.', 'bbox_head_2d.', 'conv_imitation.',
                          'norm_imitation.')

# (a key matches a prefix only up to its '.': 'backbone.' never captures 'backbone_stereo.*')
HOT_PATH_PREFIXES = ('backbone_stereo', 'feature_transformation', 'neck_3d', 'bbox_head_3d',
                     'neck', 'backbone')


def convert_liga_key(key, renames=_LIGA_HOT_PATH_RENAMES):
    """mmdet3d-style name of a LIGA-DfM ``model_state`` key.  By default only the rows for the
    keys that contain 'backbone_3d' apply; ``renames=_LIGA_RENAMES`` applies the converter's whole
    table.  Keys of the lidar teacher (``lidar_model.*``) and unmatched keys are returned
    unchanged."""
    if key.startswith('lidar_model.'):
        return key
    for old, new in renames:
        if old in key:
            return key.replace(old, new)
    return key


def _unwrap(state_dict, liga):
    if 'state_dict' in state_dict and isinstance(state_dict['state_dict'], dict):
        return state_dict['state_dict'], bool(liga)
    if 'model_state' in state_dict and isinstance(state_dict['model_state'], dict):
        return state_dict['model_state'], True
    return state_dict, bool(liga)


def hot_path_state_dicts(state_dict, liga=False):
    """Splits a detector ``state_dict`` into ``{prefix: sub_state_dict}`` for the
    hot-path modules, with the prefix stripped and the checkpoint's key order kept.
    ``liga=True`` first applies :func:`convert_liga_key` (drops ``global_step`` keys
    like the reference converter, ``:65-71``)."""
    state_dict, liga = _unwrap(state_dict, liga)
    out = {p: OrderedDict() for p in HOT_PATH_PREFIXES}
    for key, value in state_dict.items():
        if liga:
            if 'global_step' in key:
                continue
            key = convert_liga_key(key)
        for p in HOT_PATH_PREFIXES:
            if key.startswith(p + '.'):
                out[p][key[len(p) + 1:]] = value
    return out


def load_hot_path(state_dict, backbone=None, frustum=None, neck=None, strict=True,
                  liga=False, head=None, img_neck=None, img_backbone=None):
    """Loads the matching sub-dicts into the given mirror modules
    (``DfMBackbone`` / ``FrustumToVoxel`` / ``DfMNeck`` or ``OutdoorImVoxelNeck`` /
    ``Anchor3DHead``, the latter from mmdet3d-style ``bbox_head_3d.*`` keys).  ``neck`` is the
    3-D neck (``neck_3d.*``); the image neck (``neck.*``) is passed as ``img_neck``:
    DfM's ``SPPUNetNeck`` (also from LIGA ``backbone_3d.feature_neck.*``) or MultiViewDfM's
    ``FPN`` (``neck.lateral_convs.*`` / ``neck.fpn_convs.*``).  The image backbone
    (``backbone.*``: DfM's ``LIGAResNet``, also from LIGA ``backbone_3d.feature_backbone.*``, or
    MultiViewDfM's ``ResNet``, ``conv2.conv_offset.*`` of layer3 / layer4 included) is passed as
    ``img_backbone``.
    Returns the ``{prefix: load_state_dict result}`` dict."""
    parts = hot_path_state_dicts(state_dict, liga=liga)
    res = {}
    for prefix, module in (('backbone_stereo', backbone),
                           ('feature_transformation', frustum), ('neck_3d', neck),
                           ('bbox_head_3d', head), ('neck', img_neck),
                           ('backbone', img_backbone)):
        if module is None:
            continue
        if strict and not parts[prefix]:
            raise KeyError(f'checkpoint has no "{prefix}." parameters')
        res[prefix] = module.load_state_dict(parts[prefix], strict=strict)
    return res


def load_detector(ckpt, detector, liga=None):
    """Strictly loads a whole-detector checkpoint into ``modules.DfM`` / ``modules.MultiViewDfM``:
    every key of ``detector.state_dict()`` must be present (``backbone_3d.*`` included), the
    training-only entries (``TRAINING_ONLY_PREFIXES``) are skipped, and any other key the
    detector does not have raises ``KeyError``.  ``ckpt`` is a state_dict, an mmdet3d checkpoint
    (``state_dict``) or a LIGA-DfM one (``model_state``, renamed by the converter's whole table;
    ``liga=True`` applies the renames to a bare state_dict too).  Returns the sorted skipped
    keys."""
    state, liga = _unwrap(ckpt, liga)
    own = detector.state_dict()
    keep, skipped, unknown = OrderedDict(), [], []
    for key, value in state.items():
        if liga:
            if 'global_step' in key:
                continue
            key = convert_liga_key(key, _LIGA_RENAMES)
        if key.startswith(TRAINING_ONLY_PREFIXES):
            skipped.append(key)
        elif key in own:
            keep[key] = value
        else:
            unknown.append(key)
    if unknown:
        raise KeyError(f'checkpoint keys the detector does not have: {sorted(unknown)[:8]}'
                       f'{" ..." if len(unknown) > 8 else ""} ({len(unknown)} in all)')
    detector.load_state_dict(keep, strict=True)
    return sorted(skipped)


IMITATION_PREFIXES = ('conv_imitation.', 'norm_imitation.')


def load_imitation(ckpt, module, liga=None):
    """Strictly loads the imitation layers of a detector checkpoint into ``modules.DfMImitation``:
    exactly its ``conv_imitation.*`` and ``norm_imitation.*`` entries, from an mmdet3d checkpoint
    (``state_dict``), a LIGA-DfM one (``model_state``, whose ``dense_head.conv_imitation`` /
    ``dense_head.norm_imitation`` keys the converter's table renames; ``liga=True`` applies the
    renames to a bare state_dict too) or a bare state_dict.  A missing or extra imitation key
    raises.  Returns what ``load_state_dict`` returns."""
    state, liga = _unwrap(ckpt, liga)
    keep = OrderedDict()
    for key, value in state.items():
        if liga:
            if 'global_step' in key:
                continue
            key = convert_liga_key(key, _LIGA_RENAMES)
        if key.startswith(IMITATION_PREFIXES):
            keep[key] = value
    return module.load_state_dict(keep, strict=True)
