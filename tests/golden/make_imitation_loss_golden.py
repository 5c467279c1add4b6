"""Generates ``imitation_loss.npz`` in this directory by running the UNMODIFIED reference code of
DfM's LiDAR imitation loss on the CPU:

    NormalizeLayer, WeightedL2WithSigmaLoss      detectors/imitation_utils.py (whole classes,
                                                 through oracle/ref_loader.py's reference_class)
    DfM._init_imitation_layers, construct_feature_pairs, imitation_loss,
    get_imitation_reg_layer_loss                 detectors/dfm.py:213-262, 384-401, 455-539
                                                 (method source segments, extracted by ast and
                                                 executed verbatim on a holder object)

The stand-ins, stated here:

    points_in_boxes_part    mmcv 1.x's points_in_boxes_cuda_kernel.cuh rule in numpy float32,
                            every product and sum rounded on its own: cz += dz / 2; out when
                            |z - cz| > dz / 2; rotate (x - cx, y - cy) by -rz; in when strictly
                            inside +-dx / 2, +-dy / 2; the first containing box wins, -1 for none
    dist                    a single rank: get_rank() 0, all_reduce the identity
    dist_reduce_mean        the identity (models/utils/common_utils.py without a process group)
    bbox_head_3d.anchors    the reference stores ``[multi_level_anchors] * num_imgs`` (a list of
                            lists), which ``anchors[0][:, :, :, 0, 0, :3]`` cannot index; the
                            holder sets ``bbox_head_3d.anchors = [level-0 anchors of image 0]``,
                            ``modules.grid_anchors(...).reshape(1, ny, nx, 3, 2, 7)`` of the
                            shipped KITTI generator, the evident intent
    construct_feature_pairs runs with ``training = True`` (it returns nothing otherwise); the
                            eval cases put ``norm_imitation`` in eval mode before the loss

The reference runs at B = 1 only, so every case has one sample.  Inputs regenerate from the seeds
of ``synthetic.IMITATION_GOLDEN_CASES`` at the reduced grid ``IMITATION_GOLDEN_SHAPE``; the
initial scales are seeded too.  Two cases keep only the first k positive teacher rows per pair
(``synthetic.IMITATION_GOLDEN_KEEP``, ``imitation_loss_oracle.keep_positives``).  The fixture
stores per case: the in-box mask, the positive counts, the fp32 losses and scales after the call,
and the fp64 losses and autograd gradients of sum_i (1 + i / 2) loss_i with respect to both
stereo features, both conv weights and biases (fp64 stereo features and layers, the fp32
teacher and scales as the reference holds them).  Runs only where the reference tree is
available:

    python tests/golden/make_imitation_loss_golden.py
"""
import ast
import copy
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import modules, synthetic as syn  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT, reference_class  # noqa: E402
from tests import imitation_loss_oracle as O  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CFG = 'dfm_r34_1x8_kitti-3d-3class.py'
GRAD_WEIGHTS = (1.0, 1.5)


class _Dist:
    """A single rank."""
    ReduceOp = types.SimpleNamespace(SUM='sum')

    @staticmethod
    def get_rank():
        return 0

    @staticmethod
    def all_reduce(t, op=None):
        return t

    @staticmethod
    def is_available():
        return True

    @staticmethod
    def is_initialized():
        return False


def points_in_boxes_part(points, boxes):
    """mmcv's points_in_boxes_part ([B, N, 3], [B, M, 7]) -> [B, N] first box index or -1, in
    numpy float32."""
    pts = points.detach().cpu().numpy().astype(np.float32)
    bx = boxes.detach().cpu().numpy().astype(np.float32)
    out = np.full(pts.shape[:2], -1, np.int64)
    two = np.float32(2.0)
    for b in range(pts.shape[0]):
        x, y, z = pts[b, :, 0], pts[b, :, 1], pts[b, :, 2]
        for m in range(bx.shape[1] - 1, -1, -1):
            cx, cy, cz, dx, dy, dz, rz = bx[b, m]
            cz = cz + dz / two
            zout = np.abs(z - cz) > dz / two
            cosa, sina = np.cos(-rz), np.sin(-rz)
            lx = (x - cx) * cosa + (y - cy) * (-sina)
            ly = (x - cx) * sina + (y - cy) * cosa
            inside = ~zout & (lx > -dx / two) & (lx < dx / two) & (ly > -dy / two) & \
                (ly < dy / two)
            out[b, inside] = m
    return torch.from_numpy(out)


def _reference_namespace():
    ns = dict(torch=torch, nn=nn, np=np, math=math, dist=_Dist)
    rel = 'mmdet3d/models/detectors/imitation_utils.py'
    norm = reference_class(rel, 'NormalizeLayer', ns)
    l2 = reference_class(rel, 'WeightedL2WithSigmaLoss', ns)
    # the classes look `dist` up in their own globals: make sure it is the single-rank stand-in
    norm.update.__globals__['dist'] = _Dist
    ns.update(NormalizeLayer=norm, WeightedL2WithSigmaLoss=l2,
              points_in_boxes_part=points_in_boxes_part, dist_reduce_mean=lambda t: t)
    path = os.path.join(REFERENCE_ROOT, 'mmdet3d/models/detectors/dfm.py')
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == 'DfM')
    methods = {}
    for fn in cls.body:
        if isinstance(fn, ast.FunctionDef) and fn.name in (
                '_init_imitation_layers', 'construct_feature_pairs', 'imitation_loss',
                'get_imitation_reg_layer_loss'):
            code = ast.get_source_segment(src, fn)
            code = '\n'.join(l[4:] if l.startswith('    ') else l for l in code.split('\n'))
            exec(compile(code, path, 'exec'), ns)
            methods[fn.name] = ns[fn.name]
    return ns, methods


def _holder(methods, cfg, anchors, l2):
    class Holder(nn.Module):
        pass

    for k, f in methods.items():
        setattr(Holder, k, f)
    h = Holder()
    h.imitation_cfgs = cfg['imitation_cfgs']
    h.normalizer_clamp_value = cfg['normalizer_clamp_value']
    h.bbox_head_3d = types.SimpleNamespace(anchors=[anchors])
    h.loss_imitation = l2()
    h._init_imitation_layers()
    return h


def main():
    import json
    cfg = json.load(open(os.path.join(HERE, 'detector_configs.json')))[CFG]
    ag = cfg['bbox_head_3d']['anchor_generator']
    nz, ny, nx = syn.IMITATION_GOLDEN_SHAPE
    anchors = modules.grid_anchors(ag, ny, nx, 'cpu').reshape(1, ny, nx, 3, 2, 7)
    ns, methods = _reference_namespace()
    ax, ay = O.anchor_centres(ag, ny, nx)
    out = {}
    for name, (seed, num_gt, kw, training) in syn.IMITATION_GOLDEN_CASES.items():
        case = syn.make_imitation_case(seed, 1, num_gt, shape=(nz, ny, nx), **kw)
        inbox = O.inbox_mask(ax, ay, case['gt'])
        keep = syn.IMITATION_GOLDEN_KEEP.get(name)
        if keep is not None:
            O.keep_positives(case['teacher']['spatial_features_2d'], inbox, keep[0])
            O.keep_positives(case['teacher']['volume_features'], inbox, keep[1])
        g = torch.Generator().manual_seed(seed + 7)
        scales = [torch.rand((1, c), generator=g) * 1.5 + 0.5 for c in (64, 32)]
        h = _holder(methods, cfg, anchors, ns['WeightedL2WithSigmaLoss'])
        with torch.no_grad():
            for conv, w, b in zip(h.conv_imitation, case['params'][0::2], case['params'][1::2]):
                conv.weight.copy_(w.view_as(conv.weight))
                conv.bias.copy_(b)
            for key, s in zip(('spatial_features_2d', 'volume_features'), scales):
                h.norm_imitation[key].scale.copy_(s)
        gt = [types.SimpleNamespace(tensor=g_.clone()) for g_ in case['gt']]
        res = {}
        for prec in ('fp32', 'fp64'):
            hh = copy.deepcopy(h)
            st = {k: v.clone() for k, v in case['stereo'].items()}
            if prec == 'fp64':
                hh.conv_imitation.double()
                st = {k: v.double().requires_grad_() for k, v in st.items()}
            hh.train()
            raw = dict(lidar_features=case['teacher'], stereo_features=st)
            pairs = hh.construct_feature_pairs(raw)
            hh.norm_imitation.train(training)
            losses = hh.imitation_loss(pairs, gt)
            res[prec] = (hh, st, losses)
        hh, st, losses = res['fp64']
        sum(w * l for w, l in zip(GRAD_WEIGHTS, losses)).backward()
        h32, _, l32 = res['fp32']
        pos = [O.positives(inbox, case['teacher'][k]) for k in ('spatial_features_2d',
                                                               'volume_features')]
        o = dict(inbox=inbox[0].numpy().astype(np.uint8),
                 counts=np.array([int(p.sum()) for p in pos], np.int64),
                 init_scale_bev=scales[0].numpy(), init_scale_vol=scales[1].numpy(),
                 loss_fp32=np.array([float(v) for v in l32], np.float32),
                 loss_fp64=np.array([float(v) for v in losses], np.float64),
                 scale_bev=h32.norm_imitation['spatial_features_2d'].scale.numpy(),
                 scale_vol=h32.norm_imitation['volume_features'].scale.numpy(),
                 gt=case['gt'][0].numpy(), training=np.array(training))
        for i, (k, conv) in enumerate(zip(('bev', 'vol'), hh.conv_imitation)):
            src = 'spatial_features_2d' if k == 'bev' else 'volume_features'
            o[f'grad_x_{k}'] = st[src].grad.numpy()
            o[f'grad_w_{k}'] = conv.weight.grad.numpy().reshape(conv.weight.shape[0], -1)
            o[f'grad_b_{k}'] = conv.bias.grad.numpy()
        print(name, 'counts', o['counts'], 'losses', o['loss_fp32'], 'inbox', int(inbox.sum()))
        for k, v in o.items():
            out[f'{name}/{k}'] = v
    np.savez_compressed(os.path.join(HERE, 'imitation_loss.npz'), **out)


if __name__ == '__main__':
    main()
