"""Generates ``atss_loss.npz`` in this directory by running the UNMODIFIED reference code of DfM's
2-D auxiliary loss (executed verbatim as ast source segments through oracle/ref_loader.py's
``reference_class``), in fp32 on the CPU:

    LIGAATSSHead.loss_single / centerness_target / _get_target_single
                                                 dense_heads/liga_atss_head.py:176-270, 380-483
    ATSS3DCenterAssigner.assign                  core/bbox/assigners/atss_3dcenter_assigner.py

mmdet and mmcv are not in the reference tree.  The stand-ins, stated here (mmdet 2.x):

    ATSSHead.loss / get_targets / get_num_level_anchors_inside, AnchorHead.get_anchors
                                    below, as mmdet 2.x writes them: num_total_samples =
                                    max(reduce_mean(sum_b max(pos_b, 1)).item(), 1.0),
                                    bbox_avg_factor = reduce_mean(sum of the levels' centerness
                                    target sums).clamp_(min=1).item(), loss_bbox / it
    AnchorGenerator.grid_priors / valid_flags    tests/atss_loss_oracle.py's grid_priors /
                                    valid_flags: base anchor (-8 s, -8 s, 8 s, 8 s) shifted by
                                    (x s, y s) row-major; valid min(ceil(pad / s), feat) per axis
    anchor_inside_flags             allowed_border < 0: the valid flags
    unmap, images_to_levels, multi_apply, reduce_mean     mmdet's helpers (below; reduce_mean is
                                    the identity without torch.distributed)
    ATSSAssigner.__init__, AssignResult          attribute holders (below)
    BboxOverlaps2D / bbox_overlaps  anchor_loss_oracle.bbox_overlaps (mode 'iou', eps 1e-6);
                                    aligned 'giou': atss_loss_oracle.giou_aligned
    PseudoSampler                   make_anchor_loss_golden.PseudoSampler
    DeltaXYWHBBoxCoder              atss_loss_oracle.encode / decode (bbox2delta, delta2bbox with
                                    wh_ratio_clip 16 / 1000, means 0)
    FocalLoss                       make_anchor_loss_golden.FocalLoss (mmcv sigmoid_focal_loss)
    GIoULoss                        below: the zero-weight shortcut (pred * weight).sum(), else
                                    loss_weight * weight_reduce_loss(1 - giou, weight, avg_factor)
    CrossEntropyLoss(use_sigmoid)   below: binary_cross_entropy_with_logits, weight the valid mask
    weight_reduce_loss              sum / (avg_factor + FLT_EPSILON)

The two orders the reference leaves to torch (which of equal distances ``topk`` keeps at the 9th
candidate, and which of equal IoUs across GT ``max`` picks) are avoided: ``check_no_ties`` asserts
that no seeded case has either, and that no candidate's IoU lies within 1e-5 of its GT's
threshold, so the fixture does not depend on how the threshold's mean and std are rounded.

Inputs regenerate from the seeds of ``synthetic.ATSS_LOSS_GOLDEN_CASES`` at small grids of the
shipped anchor generator.  The fixture stores the per-anchor targets, the 15 loss values and the
gradients of sum_l sum_k WEIGHTS[k] (1 + l / 10) loss_k[l] with respect to the 15 head outputs.
Runs only where the reference tree is available:

    python tests/golden/make_atss_loss_golden.py
"""
import ast
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT, reference_class  # noqa: E402
from tests import anchor_loss_oracle as AO  # noqa: E402
from tests import atss_loss_oracle as O  # noqa: E402
from tests.golden.make_anchor_loss_golden import (FocalLoss, PseudoSampler, _Cfg,  # noqa: E402
                                                  images_to_levels, multi_apply,
                                                  weight_reduce_loss)

HERE = os.path.dirname(os.path.abspath(__file__))
WEIGHTS = (0.7, 1.3, 0.9)
KEYS = ('loss_cls', 'loss_bbox', 'loss_centerness')
HEAD = syn.KITTI_ATSS_HEAD
STDS = HEAD['bbox_coder']['target_stds']
STRIDES = HEAD['anchor_generator']['strides']
OBS = HEAD['anchor_generator']['octave_base_scale']


def reduce_mean(t):
    return t


def unmap(data, count, inds, fill=0):
    if data.dim() == 1:
        ret = data.new_full((count,), fill)
        ret[inds.type(torch.bool)] = data
    else:
        ret = data.new_full((count,) + data.size()[1:], fill)
        ret[inds.type(torch.bool), :] = data
    return ret


def anchor_inside_flags(flat_anchors, valid_flags, img_shape, allowed_border=0):
    assert allowed_border < 0
    return valid_flags


class AssignResult:
    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = \
            num_gts, gt_inds, max_overlaps, labels


class ATSSAssigner:
    def __init__(self, topk, iou_calculator=None, ignore_iof_thr=-1):
        self.topk, self.ignore_iof_thr = topk, ignore_iof_thr
        self.iou_calculator = lambda b1, b2, mode='iou': AO.bbox_overlaps(b1, b2)


class Coder:
    def encode(self, bboxes, gt_bboxes):
        return O.encode(bboxes, gt_bboxes, STDS)

    def decode(self, bboxes, pred_bboxes, max_shape=None):
        return O.decode(bboxes, pred_bboxes, STDS)


class GIoULoss:
    def __init__(self, eps=1e-6, loss_weight=1.0, **_):
        self.eps, self.loss_weight = eps, loss_weight

    def __call__(self, pred, target, weight=None, avg_factor=None):
        if weight is not None and not torch.any(weight > 0):
            if pred.dim() == weight.dim() + 1:
                weight = weight.unsqueeze(1)
            return (pred * weight).sum()
        loss = 1 - O.giou_aligned(pred, target, self.eps)
        return self.loss_weight * weight_reduce_loss(loss, weight, 'mean', avg_factor)


class SigmoidCrossEntropyLoss:
    def __init__(self, loss_weight=1.0, **_):
        self.loss_weight = loss_weight

    def __call__(self, pred, label, weight=None, avg_factor=None):
        valid = ((label >= 0) & (label != -100)).float()
        weight = valid if weight is None else weight * valid
        loss = torch.nn.functional.binary_cross_entropy_with_logits(pred, label.float(),
                                                                    reduction='none')
        return self.loss_weight * weight_reduce_loss(loss, weight.float(), 'mean', avg_factor)


class AnchorGenerator:
    num_levels = len(STRIDES)

    def grid_priors(self, featmap_sizes, device='cpu'):
        return O.grid_priors([tuple(s) for s in featmap_sizes], STRIDES, OBS, device)

    def valid_flags(self, featmap_sizes, pad_shape, device='cpu'):
        return O.valid_flags([tuple(s) for s in featmap_sizes], STRIDES, pad_shape, device)


# ATSSHead / AnchorHead methods of mmdet 2.x that LIGAATSSHead inherits
def get_anchors(self, featmap_sizes, img_metas, device='cpu'):
    multi_level_anchors = self.anchor_generator.grid_priors(featmap_sizes, device=device)
    anchor_list = [multi_level_anchors for _ in range(len(img_metas))]
    valid_flag_list = [self.anchor_generator.valid_flags(featmap_sizes, m['pad_shape'], device)
                       for m in img_metas]
    return anchor_list, valid_flag_list


def get_num_level_anchors_inside(self, num_level_anchors, inside_flags):
    split_inside_flags = torch.split(inside_flags, num_level_anchors)
    return [int(flags.sum()) for flags in split_inside_flags]


def get_targets(self, anchor_list, valid_flag_list, gt_bboxes_list, img_metas,
                gt_bboxes_ignore_list=None, gt_labels_list=None, label_channels=1,
                unmap_outputs=True):
    num_imgs = len(img_metas)
    num_level_anchors = [anchors.size(0) for anchors in anchor_list[0]]
    num_level_anchors_list = [num_level_anchors] * num_imgs
    for i in range(num_imgs):
        anchor_list[i] = torch.cat(anchor_list[i])
        valid_flag_list[i] = torch.cat(valid_flag_list[i])
    if gt_bboxes_ignore_list is None:
        gt_bboxes_ignore_list = [None for _ in range(num_imgs)]
    (all_anchors, all_labels, all_label_weights, all_bbox_targets, all_bbox_weights,
     pos_inds_list, neg_inds_list) = multi_apply(
        self._get_target_single, anchor_list, valid_flag_list, num_level_anchors_list,
        gt_bboxes_list, gt_bboxes_ignore_list, gt_labels_list, img_metas,
        label_channels=label_channels, unmap_outputs=unmap_outputs)
    if any([labels is None for labels in all_labels]):
        return None
    num_total_pos = sum([max(inds.numel(), 1) for inds in pos_inds_list])
    num_total_neg = sum([max(inds.numel(), 1) for inds in neg_inds_list])
    return (images_to_levels(all_anchors, num_level_anchors),
            images_to_levels(all_labels, num_level_anchors),
            images_to_levels(all_label_weights, num_level_anchors),
            images_to_levels(all_bbox_targets, num_level_anchors),
            images_to_levels(all_bbox_weights, num_level_anchors), num_total_pos, num_total_neg)


def loss(self, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas,
         gt_bboxes_ignore=None):
    featmap_sizes = [featmap.size()[-2:] for featmap in cls_scores]
    device = cls_scores[0].device
    anchor_list, valid_flag_list = self.get_anchors(featmap_sizes, img_metas, device=device)
    cls_reg_targets = self.get_targets(anchor_list, valid_flag_list, gt_bboxes, img_metas,
                                       gt_bboxes_ignore_list=gt_bboxes_ignore,
                                       gt_labels_list=gt_labels,
                                       label_channels=self.cls_out_channels)
    (anchor_list, labels_list, label_weights_list, bbox_targets_list, bbox_weights_list,
     num_total_pos, num_total_neg) = cls_reg_targets
    num_total_samples = reduce_mean(torch.tensor(num_total_pos, dtype=torch.float,
                                                 device=device)).item()
    num_total_samples = max(num_total_samples, 1.0)
    losses_cls, losses_bbox, loss_centerness, bbox_avg_factor = multi_apply(
        self.loss_single, anchor_list, cls_scores, bbox_preds, centernesses, labels_list,
        label_weights_list, bbox_targets_list, num_total_samples=num_total_samples)
    bbox_avg_factor = sum(bbox_avg_factor)
    bbox_avg_factor = reduce_mean(bbox_avg_factor).clamp_(min=1).item()
    losses_bbox = list(map(lambda x: x / bbox_avg_factor, losses_bbox))
    self.last_targets = (labels_list, label_weights_list, bbox_targets_list, bbox_weights_list,
                         num_total_pos)
    return dict(loss_cls=losses_cls, loss_bbox=losses_bbox, loss_centerness=loss_centerness)


def load():
    rel = 'mmdet3d/models/dense_heads/liga_atss_head.py'
    src = open(os.path.join(REFERENCE_ROOT, rel)).read()
    cls = [c for c in ast.parse(src).body
           if isinstance(c, ast.ClassDef) and c.name == 'LIGAATSSHead'][0]
    ns = dict(torch=torch, anchor_inside_flags=anchor_inside_flags, unmap=unmap)
    for node in cls.body:
        if isinstance(node, ast.FunctionDef) and node.name in (
                'loss_single', 'centerness_target', '_get_target_single'):
            exec(compile(ast.get_source_segment(src, node), rel, 'exec'), ns)
    assigner = reference_class('mmdet3d/core/bbox/assigners/atss_3dcenter_assigner.py',
                               'ATSS3DCenterAssigner',
                               dict(torch=torch, ATSSAssigner=ATSSAssigner,
                                    AssignResult=AssignResult))
    Head = type('LIGAATSSHead', (), dict(
        loss_single=ns['loss_single'], centerness_target=ns['centerness_target'],
        _get_target_single=ns['_get_target_single'], loss=loss, get_targets=get_targets,
        get_anchors=get_anchors, get_num_level_anchors_inside=get_num_level_anchors_inside))
    h = Head()
    h.num_classes = h.cls_out_channels = HEAD['num_classes']
    h.reg_class_agnostic, h.num_reg_channel, h.reg_avg_factor = False, 4, 'default'
    h.anchor_generator, h.bbox_coder, h.sampler = AnchorGenerator(), Coder(), PseudoSampler()
    tc = HEAD['train_cfg']
    a = dict(tc['assigner'])
    a.pop('type')
    h.assigner = assigner(**a)
    h.train_cfg = _Cfg(tc)
    h.loss_cls = FocalLoss(**HEAD['loss_cls'])
    h.loss_bbox = GIoULoss(**HEAD['loss_bbox'])
    h.loss_centerness = SigmoidCrossEntropyLoss(**HEAD['loss_centerness'])
    return h


def case_inputs(name):
    """Feature sizes, pad shapes and the case's head outputs and GT (CPU, fp32)."""
    feat_pad, pads, ngt, kw, seed = syn.ATSS_LOSS_GOLDEN_CASES[name]
    feat = syn.atss_feat_sizes(*feat_pad)
    return (feat, pads) + syn.make_atss_loss_case(seed, feat, ngt, pads, **kw)


def check_no_ties(feat, pads, gts):
    """Neither implementation-defined order nor the threshold's rounding decides a target."""
    anchors = torch.cat(O.grid_priors(feat, STRIDES, OBS))
    for pad, g in zip(pads, gts):
        if len(g) == 0:
            continue
        flags = O.valid_flags(feat, STRIDES, pad)
        a = anchors[torch.cat(flags)]
        cx, cy = (a[:, 0] + a[:, 2]) / 2.0, (a[:, 1] + a[:, 3]) / 2.0
        dx, dy = cx[:, None] - g[None, :, 4], cy[:, None] - g[None, :, 5]
        dist = (dx * dx + dy * dy).sqrt()
        ov = AO.bbox_overlaps(a, g[:, :4])
        start, cand = 0, []
        for f in flags:
            m = int(f.sum())
            d = torch.sort(dist[start:start + m], dim=0).values
            if m > O.TOPK:
                assert bool((d[O.TOPK - 1] < d[O.TOPK]).all()), 'distance tie at the 9th candidate'
            cand.append(torch.sort(dist[start:start + m], dim=0).indices[:O.TOPK] + start)
            start += m
        cand = torch.cat(cand)
        ci = ov[cand, torch.arange(len(g))]
        thr = O.threshold(ci)
        assert bool(((ci - thr[None]).abs() > 1e-5).all()), 'a candidate IoU at its threshold'
        ccx, ccy = cx[cand], cy[cand]
        e = torch.stack([ccx - g[:, 0], ccy - g[:, 1], g[:, 2] - ccx, g[:, 3] - ccy], dim=1)
        is_pos = (ci >= thr[None]) & (e.min(dim=1)[0] > 0.01)
        offered = {}
        for j, gi in zip(*torch.nonzero(is_pos, as_tuple=True)):
            offered.setdefault(int(cand[j, gi]), []).append(float(ci[j, gi]))
        for v in offered.values():
            v = sorted(v, reverse=True)
            assert len(v) == 1 or v[0] > v[1], 'equal IoU across GT'


def main():
    head = load()
    out = {}
    for name in syn.ATSS_LOSS_GOLDEN_CASES:
        feat, pads, cls, box, ctr, gts, labels = case_inputs(name)
        check_no_ties(feat, pads, gts)
        ins = [[t.clone().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
        metas = [dict(pad_shape=(h, w, 3), img_shape=(h, w, 3)) for h, w in pads]
        losses = head.loss(*ins, [g.clone() for g in gts], labels, metas)
        total = sum(WEIGHTS[k] * (1 + lv / 10) * losses[key][lv]
                    for k, key in enumerate(KEYS) for lv in range(len(feat)))
        total.backward()
        lab, lw, bt, bw, npos = head.last_targets
        lab, lw, bt, bw = (torch.cat(t, dim=1) for t in (lab, lw, bt, bw))
        # centerness targets of the positives, from the reference's own centerness_target
        anchors = torch.cat(O.grid_priors(feat, STRIDES, OBS))
        ct = torch.zeros(lab.shape)
        for b in range(len(pads)):
            pos = torch.nonzero((lab[b] >= 0) & (lab[b] < 3)).reshape(-1)
            if len(pos):
                ct[b, pos] = head.centerness_target(anchors[pos], bt[b, pos])
        for k, v in (('labels', lab), ('label_weights', lw), ('bbox_targets', bt),
                     ('bbox_weights', bw), ('centerness_targets', ct)):
            out[f'{name}.{k}'] = v.detach().numpy()
        out[f'{name}.num_total_pos'] = np.int64(npos)
        for key in KEYS:
            out[f'{name}.{key}'] = np.array([float(v.detach()) for v in losses[key]], np.float32)
        for k, ts in zip(('grad_cls', 'grad_bbox', 'grad_centerness'), ins):
            for lv, t in enumerate(ts):
                out[f'{name}.{k}.{lv}'] = t.grad.numpy()
        per_level = [int(((lab[:, a:b] >= 0) & (lab[:, a:b] < 3)).sum()) for a, b in zip(
            np.cumsum([0] + [h * w for h, w in feat])[:-1], np.cumsum([h * w for h, w in feat]))]
        print(name, 'positives per level', per_level)
    np.savez_compressed(os.path.join(HERE, 'atss_loss.npz'), **out)


if __name__ == '__main__':
    main()
