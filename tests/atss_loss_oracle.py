"""Torch restatement of DfM's 2-D auxiliary ATSS loss (``LIGAATSSHead.loss``), usable in fp32 and
fp64 on any device.

It follows, op for op, the reference's ``LIGAATSSHead.loss_single`` / ``centerness_target`` /
``_get_target_single`` (dense_heads/liga_atss_head.py:176-270, 380-483) and
``ATSS3DCenterAssigner.assign`` (core/bbox/assigners/atss_3dcenter_assigner.py:27-168), with these
restatements of the mmdet 2.x / mmcv pieces the reference imports:

    AnchorGenerator        one square anchor of side octave_base_scale * s per location at
                           (x * s, y * s), row-major; valid flags min(ceil(pad / s), feat) per axis
    anchor_inside_flags    allowed_border = -1: the valid flags
    ATSSHead.loss          num_total_samples = max(reduce_mean(sum_b max(pos_b, 1)), 1);
                           bbox_avg_factor = reduce_mean(sum of centerness targets).clamp(min=1)
    bbox_overlaps          mode 'iou' (union clamped at eps) and aligned 'giou' (eps on the union
                           and on the enclosing area)
    DeltaXYWHBBoxCoder     bbox2delta / delta2bbox, means 0, size deltas clamped to
                           +-|log(wh_ratio_clip)|
    sigmoid_focal_loss     mmcv's forward and backward (tests/anchor_loss_oracle.py)
    GIoULoss, CrossEntropyLoss(use_sigmoid=True), weight_reduce_loss
                           loss * weight, sum / (avg_factor + FLT_EPSILON), then loss_weight *

The two orders the reference leaves to torch are fixed here as the kernels fix them: equal
distances at the topk-th candidate keep the lower anchor index (a stable sort), and an anchor
positive for several GT with equal IoU goes to the first GT.  The threshold's mean and std are
formed in fp64 in candidate order (level, then distance), each rounded to fp32 and added in fp32.

Targets are computed in fp32 (``targets``): run on CUDA, they are the values the reference's fp32
ops give there.  ``losses`` takes those targets and the head outputs in any dtype.
"""
import math

import numpy as np
import torch

from tests.anchor_loss_oracle import FLT_EPS, bbox_overlaps, dist_reduce_mean, sigmoid_focal_loss

TOPK = 9


def grid_priors(feat_sizes, strides, octave_base_scale, device='cpu'):
    """AnchorGenerator.grid_priors: per level ``[H * W, 4]`` fp32 (x1, y1, x2, y2)."""
    out = []
    for (h, w), s in zip(feat_sizes, strides):
        ws = torch.tensor([float(s)]) * torch.tensor([1.0]) * torch.tensor([float(octave_base_scale)])
        base = torch.stack([0.0 - 0.5 * ws, 0.0 - 0.5 * ws, 0.0 + 0.5 * ws, 0.0 + 0.5 * ws], -1)
        sx = torch.arange(0, w, dtype=torch.float32) * s
        sy = torch.arange(0, h, dtype=torch.float32) * s
        xx, yy = sx.repeat(len(sy)), sy.view(-1, 1).repeat(1, len(sx)).view(-1)
        shifts = torch.stack([xx, yy, xx, yy], dim=-1)
        out.append((base[None] + shifts[:, None]).view(-1, 4).to(device))
    return out


def valid_flags(feat_sizes, strides, pad_shape, device='cpu'):
    """AnchorGenerator.valid_flags: per level ``[H * W]`` bool."""
    out = []
    for (h, w), s in zip(feat_sizes, strides):
        vh = min(int(np.ceil(pad_shape[0] / s)), h)
        vw = min(int(np.ceil(pad_shape[1] / s)), w)
        vx = torch.zeros(w, dtype=torch.bool)
        vy = torch.zeros(h, dtype=torch.bool)
        vx[:vw] = True
        vy[:vh] = True
        out.append((vx.repeat(h) & vy.view(-1, 1).repeat(1, w).view(-1)).to(device))
    return out


def encode(anchors, gt, stds):
    px = (anchors[..., 0] + anchors[..., 2]) * 0.5
    py = (anchors[..., 1] + anchors[..., 3]) * 0.5
    pw = anchors[..., 2] - anchors[..., 0]
    ph = anchors[..., 3] - anchors[..., 1]
    gx = (gt[..., 0] + gt[..., 2]) * 0.5
    gy = (gt[..., 1] + gt[..., 3]) * 0.5
    gw = gt[..., 2] - gt[..., 0]
    gh = gt[..., 3] - gt[..., 1]
    d = torch.stack([(gx - px) / pw, (gy - py) / ph, torch.log(gw / pw), torch.log(gh / ph)], -1)
    return d / d.new_tensor(stds)[None]


def decode(anchors, deltas, stds, wh_ratio_clip=16 / 1000):
    d = deltas * deltas.new_tensor(stds)[None]
    max_ratio = np.abs(np.log(wh_ratio_clip))
    pxy = (anchors[:, :2] + anchors[:, 2:]) * 0.5
    pwh = anchors[:, 2:] - anchors[:, :2]
    gxy = pxy + pwh * d[:, :2]
    gwh = pwh * d[:, 2:].clamp(min=-max_ratio, max=max_ratio).exp()
    return torch.cat([gxy - gwh * 0.5, gxy + gwh * 0.5], dim=-1)


def giou_aligned(b1, b2, eps=1e-6):
    """mmdet bbox_overlaps(b1, b2, mode='giou', is_aligned=True, eps)."""
    area1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    area2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt = torch.max(b1[..., :2], b2[..., :2])
    rb = torch.min(b1[..., 2:], b2[..., 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = area1 + area2 - overlap
    elt = torch.min(b1[..., :2], b2[..., :2])
    erb = torch.max(b1[..., 2:], b2[..., 2:])
    e = union.new_tensor([eps])
    union = torch.max(union, e)
    ious = overlap / union
    ewh = (erb - elt).clamp(min=0)
    earea = torch.max(ewh[..., 0] * ewh[..., 1], e)
    return ious - (earea - union) / earea


def centerness_target(anchors, bbox_targets, stds):
    gts = decode(anchors, bbox_targets, stds)
    cx = (anchors[:, 2] + anchors[:, 0]) / 2
    cy = (anchors[:, 3] + anchors[:, 1]) / 2
    lr = torch.stack([cx - gts[:, 0], gts[:, 2] - cx], dim=1)
    tb = torch.stack([cy - gts[:, 1], gts[:, 3] - cy], dim=1)
    return torch.sqrt((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) *
                      (tb.min(dim=-1)[0] / tb.max(dim=-1)[0]))


def threshold(cand_iou):
    """mean + std (unbiased) of each column of ``cand_iou`` [K, M]: both in fp64 summed in row
    order, each rounded to fp32, then added in fp32."""
    K = cand_iou.shape[0]
    c = cand_iou.double()
    s = torch.zeros_like(c[0])
    for i in range(K):
        s = s + c[i]
    mean = s / K
    v = torch.zeros_like(s)
    for i in range(K):
        d = c[i] - mean
        v = v + d * d
    return mean.float() + torch.sqrt(v / (K - 1)).float()


def atss_assign(anchors, num_level, gt, topk=TOPK):
    """ATSS3DCenterAssigner.assign over the valid anchors ``anchors`` [n, 4] (levels of
    ``num_level`` anchors each), GT [M, 6]: ``assigned`` [n] (0, or g + 1) and the thresholds [M]."""
    n, M = anchors.shape[0], gt.shape[0]
    assigned = torch.zeros(n, dtype=torch.long, device=anchors.device)
    if M == 0 or n == 0:
        return assigned, anchors.new_zeros(0)
    overlaps = bbox_overlaps(anchors, gt[:, :4])
    cx = (anchors[:, 0] + anchors[:, 2]) / 2.0
    cy = (anchors[:, 1] + anchors[:, 3]) / 2.0
    dx = cx[:, None] - gt[None, :, 4]
    dy = cy[:, None] - gt[None, :, 5]
    dist = (dx * dx + dy * dy).sqrt()
    cand, start = [], 0
    for m in num_level:
        k = min(topk, m)
        # stable: equal distances keep the lower anchor index
        order = torch.sort(dist[start:start + m], dim=0, stable=True).indices[:k]
        cand.append(order + start)
        start += m
    cand = torch.cat(cand, dim=0)                                   # [K, M]
    ar = torch.arange(M, device=anchors.device)
    cand_iou = overlaps[cand, ar]
    thr = threshold(cand_iou)
    is_pos = cand_iou >= thr[None, :]
    ccx, ccy = cx[cand], cy[cand]
    e = torch.stack([ccx - gt[:, 0], ccy - gt[:, 1], gt[:, 2] - ccx, gt[:, 3] - ccy], dim=1)
    is_pos = is_pos & (e.min(dim=1)[0] > 0.01)
    ov_inf = torch.full_like(overlaps, -math.inf)
    ov_inf[cand[is_pos], ar[None].expand_as(cand)[is_pos]] = cand_iou[is_pos]
    mx = ov_inf.max(dim=1).values
    # the first GT among equal IoUs
    arg = (ov_inf == mx[:, None]).to(torch.uint8).argmax(dim=1)
    hit = mx != -math.inf
    assigned[hit] = arg[hit] + 1
    return assigned, thr


def targets(feat_sizes, strides, octave_base_scale, gt_boxes, gt_labels, pad_shapes, cfg):
    """Per image (fp32): dict of ``assigned``, ``labels``, ``label_weights``, ``bbox_targets``
    [N, 4], ``centerness_targets`` [N] over all anchors (levels in order, row-major), ``num_pos``
    and ``thresholds`` [M]."""
    C, stds = cfg['num_classes'], cfg['target_stds']
    dev = gt_boxes[0].device if len(gt_boxes) else 'cpu'
    anchors = torch.cat(grid_priors(feat_sizes, strides, octave_base_scale, dev))
    N = anchors.shape[0]
    out = []
    for gb, gl, pad in zip(gt_boxes, gt_labels, pad_shapes):
        flags = valid_flags(feat_sizes, strides, pad, dev)
        num_level = [int(f.sum()) for f in flags]
        inside = torch.cat(flags)
        a = anchors[inside]
        asg, thr = atss_assign(a, num_level, gb.float())
        assigned = torch.zeros(N, dtype=torch.long, device=dev)
        assigned[inside] = asg
        pos = torch.nonzero(assigned > 0).reshape(-1)
        labels = torch.full((N,), C, dtype=torch.long, device=dev)
        lw = inside.float()
        bt = anchors.new_zeros(N, 4)
        ct = anchors.new_zeros(N)
        if len(pos):
            g = assigned[pos] - 1
            bt[pos] = encode(anchors[pos], gb[g, :4].float(), stds)
            labels[pos] = gl.long()[g]
            ct[pos] = centerness_target(anchors[pos], bt[pos], stds)
        out.append(dict(assigned=assigned, labels=labels, label_weights=lw, bbox_targets=bt,
                        centerness_targets=ct, num_pos=len(pos), thresholds=thr))
    return out


def losses(cls_scores, bbox_preds, centernesses, tg, feat_sizes, strides, octave_base_scale,
           cfg):
    """``dict(loss_cls=[L], loss_bbox=[L], loss_centerness=[L])`` of ``ATSSHead.loss`` with
    LIGA's ``loss_single``, from per-image targets ``tg``; the head outputs' dtype sets the
    arithmetic."""
    dt = cls_scores[0].dtype
    C, stds, w = cfg['num_classes'], cfg['target_stds'], cfg['loss_weight']
    dev = cls_scores[0].device
    anchors = grid_priors(feat_sizes, strides, octave_base_scale, dev)
    num_level = [a.shape[0] for a in anchors]
    nts = dist_reduce_mean(torch.tensor(float(sum(max(t['num_pos'], 1) for t in tg)),
                                        dtype=torch.float, device=dev)).item()
    nts = max(nts, 1.0)
    out = dict(loss_cls=[], loss_bbox=[], loss_centerness=[])
    ctr_sums, start = [], 0
    for lv, (cs, bp, cn) in enumerate(zip(cls_scores, bbox_preds, centernesses)):
        m = num_level[lv]
        sl = slice(start, start + m)
        start += m
        labels = torch.cat([t['labels'][sl] for t in tg])
        lw = torch.cat([t['label_weights'][sl] for t in tg]).to(dt)
        btg = torch.cat([t['bbox_targets'][sl] for t in tg]).to(dt)
        ctg = torch.cat([t['centerness_targets'][sl] for t in tg])
        an = anchors[lv].to(dt).repeat(len(tg), 1)
        cls = cs.permute(0, 2, 3, 1).reshape(-1, C)
        out['loss_cls'].append(w[0] * ((sigmoid_focal_loss(cls, labels, cfg['gamma'],
                                                           cfg['alpha']) * lw[:, None]).sum() /
                                       (nts + FLT_EPS)))
        reg = bp.permute(0, 2, 3, 1).reshape(-1, 4, C)
        reg = torch.cat([reg, torch.zeros_like(reg[:, :, :1])], dim=-1)
        reg = torch.gather(reg, 2, labels.reshape(-1, 1, 1).repeat(1, 4, 1)).squeeze(-1)
        ctr = cn.permute(0, 2, 3, 1).reshape(-1)
        pos = torch.nonzero((labels >= 0) & (labels < C)).reshape(-1)
        if len(pos):
            ct = ctg[pos].to(dt)
            pb = decode(an[pos], reg[pos], stds)
            tb = decode(an[pos], btg[pos], stds)
            if not bool((ct > 0).any()):
                lb = (pb * ct[:, None]).sum()                    # GIoULoss's zero-weight shortcut
            else:
                lb = w[1] * (((1 - giou_aligned(pb, tb, cfg['giou_eps'])) * ct).sum() /
                             (1.0 + FLT_EPS))
            bce = torch.nn.functional.binary_cross_entropy_with_logits(ctr[pos], ct,
                                                                       reduction='none')
            lc = w[2] * (bce.sum() / (nts + FLT_EPS))
            ctr_sums.append(ctg[pos].sum())
        else:
            lb = bp.sum() * 0
            lc = cn.sum() * 0
            ctr_sums.append(ctg.new_tensor(0.))
        out['loss_bbox'].append(lb)
        out['loss_centerness'].append(lc)
    baf = sum(ctr_sums)
    baf = dist_reduce_mean(baf).clamp_(min=1).item()
    out['loss_bbox'] = [x / baf for x in out['loss_bbox']]
    return out
