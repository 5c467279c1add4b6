"""Generates ``anchor_loss.npz`` in this directory by running the UNMODIFIED reference code of the
anchor heads' training loss (executed verbatim as ast source segments through
oracle/ref_loader.py's ``reference_class`` / ``reference_function``), in fp32 on the CPU:

    AnchorTrainMixin.anchor_target_3d / _single / anchor_target_single_assigner,
    get_direction_target                             dense_heads/train_mixins.py
    Anchor3DHead.get_anchors / loss / loss_single / add_sin_difference
                                                     dense_heads/anchor3d_head.py:179-406
    LIGAAnchor3DHead.get_anchors / loss_single       dense_heads/liga_anchor3d_head.py:80-226
    dist_reduce_mean                                 models/utils/common_utils.py
    iou3d_loss, IOU3DLoss                            models/losses/iou3d_loss.py
    DeltaXYZWLHRBBoxCoder                            core/bbox/coders/delta_xyzwhlr_bbox_coder.py
    bbox_overlaps_nearest_3d                         core/bbox/iou_calculators/iou3d_calculator.py
    BaseInstance3DBoxes.nearest_bev, LiDARInstance3DBoxes, limit_period
    Anchor3DRangeGenerator, AlignedAnchor3DRangeGenerator

mmdet and mmcv are not in the reference tree.  The stand-ins, stated here:

    MaxIoUAssigner, bbox_overlaps     tests/anchor_loss_oracle.py's max_iou_assign / bbox_overlaps
    PseudoSampler                     positives gt_inds > 0, negatives gt_inds == 0 (below)
    multi_apply, images_to_levels     mmdet's two helpers (below)
    FocalLoss, SmoothL1Loss, CrossEntropyLoss, weighted_loss / weight_reduce_loss
                                      mmdet 2.x forms (below): loss * weight, then
                                      sum / (avg_factor + FLT_EPSILON), then loss_weight *
    sigmoid_focal_loss                mmcv's forward / backward: anchor_loss_oracle._FocalFn
    diff_iou_rotated_3d               anchor_loss_oracle.diff_iou_rotated_3d

Inputs regenerate from the seeds of ``synthetic.ANCHOR_LOSS_GOLDEN_CASES`` (small grids of the
shipped anchor generators; the fixture stores per-anchor targets, loss values and the gradients
of sum_k WEIGHTS[k] * loss_k with respect to the three head outputs).  LIGA cases where the
reference's ``loss_iou`` cannot run (no positive, or batch > 1) run it without ``loss_iou``.
Runs only where the reference tree is available:

    python tests/golden/make_anchor_loss_golden.py
"""
import ast
import os
import sys
import warnings
from abc import abstractmethod
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT, reference_class, reference_function  # noqa: E402
from tests import anchor_loss_oracle as O  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
WEIGHTS = (0.7, 1.3, 0.9, 1.1)


class _Cfg(dict):
    """mmcv ConfigDict's attribute access."""
    __getattr__ = dict.__getitem__


def multi_apply(func, *args, **kwargs):
    res = map(partial(func, **kwargs) if kwargs else func, *args)
    return tuple(map(list, zip(*res)))


def images_to_levels(target, num_levels):
    target = torch.stack(target, 0)
    out, start = [], 0
    for n in num_levels:
        out.append(target[:, start:start + n])
        start += n
    return out


def weight_reduce_loss(loss, weight=None, reduction='mean', avg_factor=None):
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        return loss.mean() if reduction == 'mean' else (loss.sum() if reduction == 'sum' else loss)
    assert reduction == 'mean'
    return loss.sum() / (avg_factor + torch.finfo(torch.float32).eps)


def weighted_loss(fn):
    def wrapper(pred, target, weight=None, reduction='mean', avg_factor=None, **kwargs):
        return weight_reduce_loss(fn(pred, target, **kwargs), weight, reduction, avg_factor)
    return wrapper


class FocalLoss:
    def __init__(self, gamma=2.0, alpha=0.25, loss_weight=1.0, **_):
        self.gamma, self.alpha, self.loss_weight = gamma, alpha, loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        loss = O.sigmoid_focal_loss(pred.contiguous(), target.contiguous(), self.gamma,
                                    self.alpha)
        if weight is not None and weight.shape != loss.shape:
            weight = weight.view(-1, 1)
        return self.loss_weight * weight_reduce_loss(loss, weight, 'mean', avg_factor)


class SmoothL1Loss:
    def __init__(self, beta=1.0, loss_weight=1.0, **_):
        self.beta, self.loss_weight = beta, loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        diff = torch.abs(pred - target)
        loss = torch.where(diff < self.beta, 0.5 * diff * diff / self.beta,
                           diff - 0.5 * self.beta)
        return self.loss_weight * weight_reduce_loss(loss, weight, 'mean', avg_factor)


class CrossEntropyLoss:
    def __init__(self, loss_weight=1.0, **_):
        self.loss_weight = loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        loss = torch.nn.functional.cross_entropy(pred, target, reduction='none')
        return self.loss_weight * weight_reduce_loss(loss, weight.float(), 'mean', avg_factor)


class PseudoSampler:
    def sample(self, assign_result, bboxes, gt_bboxes):
        r = _Cfg()
        r['pos_inds'] = torch.nonzero(assign_result.gt_inds > 0, as_tuple=False).squeeze(-1)\
            .unique()
        r['neg_inds'] = torch.nonzero(assign_result.gt_inds == 0, as_tuple=False).squeeze(-1)\
            .unique()
        r['pos_bboxes'] = bboxes[r['pos_inds']]
        r['pos_assigned_gt_inds'] = assign_result.gt_inds[r['pos_inds']] - 1
        r['pos_gt_bboxes'] = gt_bboxes[r['pos_assigned_gt_inds'], :]
        return r


def load():
    u = 'mmdet3d/core/bbox/structures/utils.py'
    limit_period = reference_function(u, 'limit_period', dict(torch=torch, np=np))
    mmcv = type('mmcv', (), {'is_list_of': staticmethod(
        lambda seq, t: isinstance(seq, list) and all(isinstance(s, t) for s in seq))})
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
    overlaps = reference_function('mmdet3d/core/bbox/iou_calculators/iou3d_calculator.py',
                                  'bbox_overlaps_nearest_3d',
                                  dict(torch=torch, get_box_type=lambda c: (lidar, None),
                                       bbox_overlaps=lambda a, b, mode='iou', is_aligned=False:
                                       O.bbox_overlaps(a, b)))
    tm = 'mmdet3d/models/dense_heads/train_mixins.py'
    dir_target = reference_function(tm, 'get_direction_target',
                                     dict(torch=torch, np=np, limit_period=limit_period))
    mixin = reference_class(tm, 'AnchorTrainMixin',
                            dict(torch=torch, np=np, limit_period=limit_period,
                                 images_to_levels=images_to_levels, multi_apply=multi_apply,
                                 get_direction_target=dir_target))
    reduce_mean = reference_function('mmdet3d/models/utils/common_utils.py', 'dist_reduce_mean',
                                     dict(torch=torch, dist=torch.distributed))
    il = 'mmdet3d/models/losses/iou3d_loss.py'
    iou3d_loss = weighted_loss(reference_function(
        il, 'iou3d_loss', dict(torch=torch, diff_iou_rotated_3d=lambda a, b:
                               O.diff_iou_rotated_3d(a[0], b[0])[None])))
    iou_cls = reference_class(il, 'IOU3DLoss', dict(torch=torch, nn=torch.nn,
                                                    iou3d_loss=iou3d_loss))

    def methods(rel, cname, names, ns):
        src = open(os.path.join(REFERENCE_ROOT, rel)).read()
        cls = [c for c in ast.parse(src).body
               if isinstance(c, ast.ClassDef) and c.name == cname][0]
        ns = dict(ns)
        for node in cls.body:
            if isinstance(node, ast.FunctionDef) and node.name in names:
                keep = [d for d in node.decorator_list
                        if isinstance(d, ast.Name) and d.id == 'staticmethod']
                node.decorator_list = keep
                exec(compile(ast.Module(body=[node], type_ignores=[]), rel, 'exec'), ns)
        return {n: ns[n] for n in names}

    base_ns = dict(torch=torch, np=np, multi_apply=multi_apply)
    a3d = methods('mmdet3d/models/dense_heads/anchor3d_head.py', 'Anchor3DHead',
                  ('get_anchors', 'loss', 'loss_single', 'add_sin_difference'), base_ns)
    liga = methods('mmdet3d/models/dense_heads/liga_anchor3d_head.py', 'LIGAAnchor3DHead',
                   ('get_anchors', 'loss_single'), dict(base_ns, dist_reduce_mean=reduce_mean))

    class Assigner:
        """MaxIoUAssigner stand-in with BboxOverlapsNearest3D (gt first)."""

        def __init__(self, cfg):
            self.thr = (cfg['pos_iou_thr'], cfg['neg_iou_thr'], cfg['min_pos_iou'])

        def assign(self, bboxes, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None):
            r = _Cfg()
            r['gt_inds'] = O.max_iou_assign(overlaps(gt_bboxes, bboxes), *self.thr)
            return r

    def make_head(kind, cfg):
        is_liga = kind == 'liga'
        ns = dict(a3d, **(liga if is_liga else {}))
        Head = type('Head', (mixin,), ns)
        h = Head()
        gcfg = dict(cfg['generator'])
        k = gcfg.pop('type')
        h.anchor_generator = (agen if k == 'AlignedAnchor3DRangeGenerator' else gen)(**gcfg)
        h.box_code_size, h.num_classes, h.use_sigmoid_cls, h.sampling = 7, 3, True, False
        h.num_anchors = 6
        h.cls_out_channels = h.num_anchors * h.num_classes
        h.use_direction_classifier = True
        h.bbox_coder, h.bbox_sampler = coder(), PseudoSampler()
        h.train_cfg = _Cfg(cfg['train_cfg'])
        h.bbox_assigner = [Assigner(a) for a in cfg['train_cfg']['assigner']]
        h.assign_per_class, h.diff_rad_by_sin = cfg['assign_per_class'], True
        h.dir_offset, h.dir_limit_offset = cfg['dir_offset'], 0
        losses = cfg['losses']
        h.loss_cls = FocalLoss(**losses['loss_cls'])
        h.loss_bbox = SmoothL1Loss(**losses['loss_bbox'])
        h.loss_dir = CrossEntropyLoss(**losses['loss_dir'])
        li = losses.get('loss_iou') if cfg['with_iou'] else None
        h.loss_iou = iou_cls(loss_weight=li['loss_weight']) if li else None
        h.normalizer_clamp_value, h.reduce_avg_factor = 10, True
        return h

    return make_head


def case_config(name):
    kind, ny, nx, ngt, kw, with_iou, seed = syn.ANCHOR_LOSS_GOLDEN_CASES[name]
    if kind == 'liga':
        cfg = dict(generator=syn.KITTI_ANCHOR_GENERATOR, train_cfg=syn.KITTI_TRAIN_CFG,
                   losses=syn.KITTI_LOSSES, assign_per_class=True,
                   dir_offset=syn.KITTI_DIR_OFFSET, with_iou=with_iou)
    else:
        cfg = dict(generator=syn.WAYMO_ANCHOR_GENERATOR, train_cfg=syn.WAYMO_TRAIN_CFG,
                   losses=syn.WAYMO_LOSSES, assign_per_class=False,
                   dir_offset=syn.WAYMO_DIR_OFFSET, with_iou=False)
    return kind, ny, nx, ngt, kw, seed, cfg


def case_inputs(name):
    """Head outputs and GT of a golden case, from its seed (CPU, fp32)."""
    kind, ny, nx, ngt, kw, seed, cfg = case_config(name)
    anchors = modules.grid_anchors(cfg['generator'], ny, nx, 'cpu')
    return (anchors,) + syn.make_anchor_loss_case(seed, anchors.numpy(), ny, nx, 3, 2, 3, ngt,
                                                  **kw)


def main():
    make_head = load()
    out = {}
    for name in syn.ANCHOR_LOSS_GOLDEN_CASES:
        kind, ny, nx, ngt, kw, seed, cfg = case_config(name)
        head = make_head(kind, cfg)
        anchors, cls, box, dirc, gts, labels = case_inputs(name)
        ref_anchors = head.anchor_generator.grid_anchors([(ny, nx)], device='cpu')[0]
        assert torch.equal(ref_anchors.reshape(-1, 7), anchors)
        ins = [t.clone().requires_grad_() for t in (cls, box, dirc)]
        metas = [{} for _ in ngt]
        # the targets as loss() computes them, kept for the fixture
        tgt = head.anchor_target_3d(
            head.get_anchors([(ny, nx)], metas, device='cpu'), [g.clone() for g in gts], metas,
            gt_labels_list=labels, num_classes=3, label_channels=18, sampling=False)
        losses = head.loss([ins[0]], [ins[1]], [ins[2]], [g.clone() for g in gts], labels, metas)
        keys = ['loss_cls', 'loss_bbox', 'loss_dir'] + (['loss_iou'] if head.loss_iou else [])
        total = sum(w * losses[k][0] for w, k in zip(WEIGHTS, keys))
        total.backward()
        for i, k in enumerate(('labels', 'label_weights', 'bbox_targets', 'bbox_weights',
                               'dir_targets', 'dir_weights')):
            out[f'{name}.{k}'] = tgt[i][0].numpy()
        out[f'{name}.num_total_pos'] = np.int64(tgt[6])
        for k in keys:
            out[f'{name}.{k}'] = np.float32(losses[k][0].item())
        for k, t in zip(('grad_cls', 'grad_bbox', 'grad_dir'), ins):
            out[f'{name}.{k}'] = t.grad.numpy()
        npos = int(((tgt[0][0] >= 0) & (tgt[0][0] < 3)).sum())
        print(name, 'positives', npos, {k: float(losses[k][0]) for k in keys})
    np.savez_compressed(os.path.join(HERE, 'anchor_loss.npz'), **out)


if __name__ == '__main__':
    main()
