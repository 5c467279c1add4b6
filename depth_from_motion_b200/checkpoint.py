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

# (old substring, new substring), in the reference's matching order for the keys that
# contain 'backbone_3d' (convert_dfm_checkpoints.py:49-53)
_LIGA_RENAMES = (
    ('backbone_3d.feature_backbone', 'backbone'),
    ('backbone_3d.feature_neck', 'neck'),
    ('backbone_3d.sem_neck', 'neck_2d'),
    ('backbone_3d.rpn3d_convs', 'feature_transformation.voxel_convs'),
    ('backbone_3d', 'backbone_stereo'),
)

# (a key matches a prefix only up to its '.': 'backbone.' never captures 'backbone_stereo.*')
HOT_PATH_PREFIXES = ('backbone_stereo', 'feature_transformation', 'neck_3d', 'bbox_head_3d',
                     'neck', 'backbone')


def convert_liga_key(key):
    """mmdet3d-style name of a LIGA-DfM ``model_state`` key, for the prefixes that
    involve the hot path; keys of the lidar teacher (``lidar_model.*``) and of other
    modules are returned unchanged."""
    if key.startswith('lidar_model.'):
        return key
    for old, new in _LIGA_RENAMES:
        if old in key:
            return key.replace(old, new)
    return key


def hot_path_state_dicts(state_dict, liga=False):
    """Splits a detector ``state_dict`` into ``{prefix: sub_state_dict}`` for the
    hot-path modules, with the prefix stripped and the checkpoint's key order kept.
    ``liga=True`` first applies :func:`convert_liga_key` (drops ``global_step`` keys
    like the reference converter, ``:65-71``)."""
    if 'state_dict' in state_dict and isinstance(state_dict['state_dict'], dict):
        state_dict = state_dict['state_dict']
    elif 'model_state' in state_dict and isinstance(state_dict['model_state'], dict):
        state_dict, liga = state_dict['model_state'], True
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
