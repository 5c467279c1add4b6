"""Generates ``box_post.npz`` in this directory by running the UNMODIFIED reference code of the
anchor heads' ``get_bboxes`` (executed verbatim as ast source segments through
oracle/ref_loader.py's ``reference_class`` / ``reference_function``):

    Anchor3DHead.get_bboxes / get_bboxes_single     dense_heads/anchor3d_head.py:407-547
    Anchor3DRangeGenerator, AlignedAnchor3DRangeGenerator   core/anchor/anchor_3d_generator.py
    DeltaXYZWLHRBBoxCoder.decode                     core/bbox/coders/delta_xyzwhlr_bbox_coder.py
    xywhr2xyxyr, limit_period                         core/bbox/structures/utils.py
    BaseInstance3DBoxes, LiDARInstance3DBoxes         core/bbox/structures/
    box3d_multiclass_nms, nms_bev                     core/post_processing/box3d_nms.py

mmcv's ``nms_rotated`` is not in the reference tree; the only stand-in is
``tests/box_post_oracle.py``'s fp64 restatement (see its docstring for the corner convention).
Two mmcv utilities the constructors touch are given trivial forms: ``mmcv.is_list_of`` and a
dict with attribute access for the test config.  Inputs regenerate from the seeds of
``synthetic.BOX_POST_CASES``; the fixture stores the reference outputs, the anchor tables,
input checksums and SHA-256 digests of the anchor tables at the shipped grids.  Runs only where
the reference tree is available:

    python tests/golden/make_box_post_golden.py
"""
import ast
import hashlib
import os
import sys
import warnings
from abc import abstractmethod

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT, reference_class, reference_function  # noqa: E402
from tests import box_post_oracle as BP  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


class _Cfg(dict):
    """mmcv ConfigDict's attribute access."""
    __getattr__ = dict.__getitem__


def _nms_rotated(dets, scores, iou_threshold):
    """mmcv.ops.nms_rotated stand-in: (dets[keep], keep) with keep in score order."""
    order = torch.argsort(scores, descending=True, stable=True)
    keep = order[BP.nms_rotated(dets[order], iou_threshold)]
    return dets[keep], keep


def _is_list_of(seq, t):
    return isinstance(seq, list) and all(isinstance(s, t) for s in seq)


def load():
    mmcv = type('mmcv', (), {'is_list_of': staticmethod(_is_list_of)})
    u = 'mmdet3d/core/bbox/structures/utils.py'
    limit_period = reference_function(u, 'limit_period', dict(torch=torch, np=np))
    xywhr2xyxyr = reference_function(u, 'xywhr2xyxyr', dict(torch=torch, np=np))
    g = 'mmdet3d/core/anchor/anchor_3d_generator.py'
    gen = reference_class(g, 'Anchor3DRangeGenerator', dict(torch=torch, mmcv=mmcv))
    agen = reference_class(g, 'AlignedAnchor3DRangeGenerator',
                           dict(torch=torch, mmcv=mmcv, Anchor3DRangeGenerator=gen))
    coder = reference_class('mmdet3d/core/bbox/coders/delta_xyzwhlr_bbox_coder.py',
                            'DeltaXYZWLHRBBoxCoder', dict(torch=torch, BaseBBoxCoder=object))
    base = reference_class('mmdet3d/core/bbox/structures/base_box3d.py', 'BaseInstance3DBoxes',
                           dict(torch=torch, np=np, warnings=warnings,
                                abstractmethod=abstractmethod, limit_period=limit_period))
    lidar = reference_class('mmdet3d/core/bbox/structures/lidar_box3d.py',
                            'LiDARInstance3DBoxes',
                            dict(torch=torch, np=np, BaseInstance3DBoxes=base))
    n = 'mmdet3d/core/post_processing/box3d_nms.py'
    nms_bev = reference_function(n, 'nms_bev', dict(torch=torch, nms_rotated=_nms_rotated))
    multiclass = reference_function(n, 'box3d_multiclass_nms',
                                    dict(torch=torch, nms_bev=nms_bev, nms_normal_bev=None))
    rel = 'mmdet3d/models/dense_heads/anchor3d_head.py'
    src = open(os.path.join(REFERENCE_ROOT, rel)).read()
    cls = [c for c in ast.parse(src).body
           if isinstance(c, ast.ClassDef) and c.name == 'Anchor3DHead'][0]
    ns = dict(torch=torch, np=np, box3d_multiclass_nms=multiclass, xywhr2xyxyr=xywhr2xyxyr,
              limit_period=limit_period)
    for node in cls.body:
        if isinstance(node, ast.FunctionDef) and node.name in ('get_bboxes', 'get_bboxes_single'):
            node.decorator_list = []
            exec(compile(ast.Module(body=[node], type_ignores=[]), rel, 'exec'), ns)

    class Head:
        """Attribute holder: what Anchor3DHead.__init__ sets that get_bboxes reads."""

        def __init__(self, generator, num_classes, use_sigmoid, test_cfg, dir_offset):
            g = dict(generator)
            kind = g.pop('type')
            self.anchor_generator = (agen if kind == 'AlignedAnchor3DRangeGenerator' else gen)(**g)
            self.box_code_size = 7
            self.use_sigmoid_cls = use_sigmoid
            self.num_classes = num_classes if use_sigmoid else num_classes + 1
            self.bbox_coder = coder()
            self.test_cfg = _Cfg(test_cfg)
            self.dir_offset, self.dir_limit_offset = dir_offset, 0

        get_bboxes = ns['get_bboxes']
        get_bboxes_single = ns['get_bboxes_single']

    return Head, lidar


def main():
    Head, lidar = load()
    out = {}
    for name, (generator, ny, nx, cfg, sigmoid, dir_offset, seed, kw) in \
            syn.BOX_POST_CASES.items():
        cls, box, dirc = syn.make_box_post_case(seed, ny, nx, **kw)
        head = Head(generator, 3, sigmoid, cfg, dir_offset)
        anchors = head.anchor_generator.grid_anchors([(ny, nx)], device='cpu')[0].reshape(-1, 7)
        with torch.no_grad():
            (boxes, scores, labels), = head.get_bboxes([cls[None]], [box[None]], [dirc[None]],
                                                       [dict(box_type_3d=lidar)])
        assert isinstance(boxes, lidar)
        out[f'{name}.boxes'] = boxes.tensor.numpy()
        out[f'{name}.scores'] = scores.numpy()
        out[f'{name}.labels'] = labels.numpy()
        out[f'{name}.anchors'] = anchors.numpy()
        out[f'{name}.input_sum'] = np.float64(sum(t.double().abs().sum().item()
                                                  for t in (cls, box, dirc)))
        print(name, tuple(boxes.tensor.shape), np.bincount(labels.numpy(), minlength=3))
    # anchor tables at the shipped grids (KITTI 304 x 288, Waymo 300 x 220): digests only
    for name, generator, ny, nx in (('kitti', syn.KITTI_ANCHOR_GENERATOR, 304, 288),
                                    ('waymo', syn.WAYMO_ANCHOR_GENERATOR, 300, 220)):
        a = Head(generator, 3, True, syn.KITTI_TEST_CFG, 0.0).anchor_generator.grid_anchors(
            [(ny, nx)], device='cpu')[0].reshape(-1, 7).contiguous()
        out[f'{name}_full.anchors_sha256'] = np.array(hashlib.sha256(a.numpy().tobytes())
                                                      .hexdigest())
        out[f'{name}_full.shape'] = np.array(a.shape)
    np.savez_compressed(os.path.join(HERE, 'box_post.npz'), **out)


if __name__ == '__main__':
    main()
