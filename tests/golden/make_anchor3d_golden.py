"""Generates ``anchor3d_head.npz`` in this directory from the UNMODIFIED reference source:
``Anchor3DHead._init_layers`` and ``forward_single``
(mmdet3d/models/dense_heads/anchor3d_head.py:139-164) are executed verbatim (ast source
segments, the way oracle/ref_loader.py builds its LIGAAnchor3DHead holder) on an attribute
holder configured like the ``bbox_head_3d`` of the shipped Waymo configs
(configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync[_10sweeps].py:35-67).
Runs only where the reference tree is available:

    python tests/golden/make_anchor3d_golden.py

Inputs regenerate from the seed (``synthetic.make_anchor3d_head_case``): a non-negative
synthetic BEV map with 256 channels on a 37 x 29 grid (1,073 cells, i.e. 8 full 128-cell tiles of
the tensor-core kernel plus a ragged tail of 49) and random weights and biases (not the
near-zero init), so every output carries signal.  The fixture stores the reference outputs,
checksums of the inputs, and the reference ``state_dict`` keys and shapes.
"""
import ast
import os
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
NUM_CLASSES, NUM_ANCHORS, BOX_CODE_SIZE = 3, 6, 7   # 3 sizes x 2 rotations, DeltaXYZWLHR


def reference_head_class(feat):
    rel = 'mmdet3d/models/dense_heads/anchor3d_head.py'
    src = open(os.path.join(REFERENCE_ROOT, rel)).read()
    cls = [n for n in ast.parse(src).body
           if isinstance(n, ast.ClassDef) and n.name == 'Anchor3DHead'][0]
    ns = dict(torch=torch, nn=nn)
    for node in cls.body:
        if isinstance(node, ast.FunctionDef) and node.name in ('_init_layers', 'forward_single'):
            exec(compile(ast.get_source_segment(src, node), rel, 'exec'), ns)

    class Anchor3DHead(nn.Module):
        """Attribute holder: what Anchor3DHead.__init__ sets before `_init_layers()`
        (anchor3d_head.py:73-112)."""

        def __init__(self):
            super().__init__()
            self.num_classes, self.feat_channels = NUM_CLASSES, feat
            self.num_anchors, self.box_code_size = NUM_ANCHORS, BOX_CODE_SIZE
            self.use_direction_classifier = True
            self._init_layers()

        _init_layers = ns['_init_layers']
        forward_single = ns['forward_single']

    return Anchor3DHead


def main():
    case = syn.ANCHOR3D_HEAD_CASE
    x, sd = syn.make_anchor3d_head_case(**case)
    head = reference_head_class(case['feat'])().eval()
    head.load_state_dict(sd, strict=True)
    with torch.no_grad():
        cls, box, dirc = head.forward_single(x)
    keys = [k for k in head.state_dict()]
    shapes = np.array([','.join(str(n) for n in v.shape) for v in head.state_dict().values()])
    np.savez_compressed(
        os.path.join(HERE, 'anchor3d_head.npz'),
        cls_score=cls.numpy(), bbox_pred=box.numpy(), dir_cls_preds=dirc.numpy(),
        state_keys=np.array(keys), state_shapes=shapes,
        x_sum=np.float64(x.double().sum().item()), x_abs=np.float64(x.double().abs().sum().item()),
        w_abs=np.float64(sum(v.double().abs().sum().item() for v in sd.values())))
    print('anchor3d_head', tuple(cls.shape), tuple(box.shape), tuple(dirc.shape),
          float(box.abs().max()))


if __name__ == '__main__':
    main()
