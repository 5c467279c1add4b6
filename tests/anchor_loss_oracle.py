"""Torch restatement of the anchor heads' training loss, usable in fp32 and fp64 on any device.

It follows, op for op, the reference's ``AnchorTrainMixin`` (dense_heads/train_mixins.py:102-350),
``Anchor3DHead.loss`` / ``loss_single`` / ``add_sin_difference`` (anchor3d_head.py:199-406),
``LIGAAnchor3DHead.loss_single`` (liga_anchor3d_head.py:130-226), ``DeltaXYZWLHRBBoxCoder``,
``bbox_overlaps_nearest_3d`` / ``nearest_bev`` / ``limit_period`` and ``iou3d_loss``, with these
restatements of the mmdet 2.x / mmcv pieces the reference imports:

    bbox_overlaps          mmdet, mode 'iou': union = max(area1 + area2 - overlap, 1e-6)
    MaxIoUAssigner         thresholds, per-anchor argmax (first GT on ties), low-quality pass
                           with gt_max_assign_all (GT in index order, later ones win)
    PseudoSampler          positives assigned > 0, negatives assigned == 0
    sigmoid_focal_loss     mmcv's forward and backward formulas, FLT_MIN clamp inside both logs
    SmoothL1Loss, CrossEntropyLoss, weight_reduce_loss   sum / (avg_factor + FLT_EPSILON)
    diff_iou_rotated_3d    mmcv's vertex set (corners inside, edge crossings), angle sort and
                           shoelace area; the 7-vector's z read as the box centre

Targets are computed in fp32 (``targets``): run on CUDA, they are the values the reference's
fp32 ops give there.  ``losses`` takes those targets and the head outputs in any dtype.
"""
import numpy as np
import torch

FLT_MIN = float(np.finfo(np.float32).tiny)
FLT_EPS = float(np.finfo(np.float32).eps)


def limit_period(val, offset=0.5, period=np.pi):
    return val - torch.floor(val / period + offset) * period


def nearest_bev(boxes):
    bev = boxes[:, [0, 1, 3, 4, 6]]
    normed = torch.abs(limit_period(bev[:, -1], 0.5, np.pi))
    cond = (normed > np.pi / 4)[..., None]
    xywh = torch.where(cond, bev[:, [0, 1, 3, 2]], bev[:, :4])
    centers, dims = xywh[:, :2], xywh[:, 2:]
    return torch.cat([centers - dims / 2, centers + dims / 2], dim=-1)


def bbox_overlaps(b1, b2, eps=1e-6):
    area1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    area2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt = torch.max(b1[..., :, None, :2], b2[..., None, :, :2])
    rb = torch.min(b1[..., :, None, 2:], b2[..., None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = area1[..., None] + area2[..., None, :] - overlap
    union = torch.max(union, union.new_tensor([eps]))
    return overlap / union


def max_iou_assign(overlaps, pos_thr, neg_thr, min_pos):
    """``assigned`` per anchor: -1 ignored, 0 negative, i + 1 for GT row i of ``overlaps``."""
    G, N = overlaps.shape
    assigned = overlaps.new_full((N,), -1, dtype=torch.long)
    if G == 0:
        return assigned.zero_()
    max_ov, argmax_ov = overlaps.max(dim=0)
    # torch.max returns the first maximum on CPU; state it so the device does not matter
    argmax_ov = (overlaps == max_ov[None]).to(torch.uint8).argmax(dim=0)
    gt_max = overlaps.max(dim=1).values
    assigned[(max_ov >= 0) & (max_ov < neg_thr)] = 0
    pos = max_ov >= pos_thr
    assigned[pos] = argmax_ov[pos] + 1
    for i in range(G):
        if gt_max[i] >= min_pos:
            assigned[overlaps[i] == gt_max[i]] = i + 1
    return assigned


def encode(src, dst):
    xa, ya, za, wa, la, ha, ra = torch.split(src, 1, dim=-1)
    xg, yg, zg, wg, lg, hg, rg = torch.split(dst, 1, dim=-1)
    za = za + ha / 2
    zg = zg + hg / 2
    diagonal = torch.sqrt(la**2 + wa**2)
    return torch.cat([(xg - xa) / diagonal, (yg - ya) / diagonal, (zg - za) / ha,
                      torch.log(wg / wa), torch.log(lg / la), torch.log(hg / ha), rg - ra], dim=-1)


def decode(anchors, deltas):
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, wt, lt, ht, rt = torch.split(deltas, 1, dim=-1)
    za = za + ha / 2
    diagonal = torch.sqrt(la**2 + wa**2)
    xg = xt * diagonal + xa
    yg = yt * diagonal + ya
    zg = zt * ha + za
    lg = torch.exp(lt) * la
    wg = torch.exp(wt) * wa
    hg = torch.exp(ht) * ha
    rg = rt + ra
    zg = zg - hg / 2
    return torch.cat([xg, yg, zg, wg, lg, hg, rg], dim=-1)


def direction_target(anchors, reg_targets, dir_offset, dir_limit_offset, num_bins=2):
    rot_gt = reg_targets[..., 6] + anchors[..., 6]
    offset_rot = limit_period(rot_gt - dir_offset, dir_limit_offset, 2 * np.pi)
    t = torch.floor(offset_rot / (2 * np.pi / num_bins)).long()
    return torch.clamp(t, min=0, max=num_bins - 1)


def targets(anchors, num_sizes, num_rots, gt_boxes, gt_labels, cfg):
    """Per sample (fp32): dict of ``assigned`` (g + 1 indexes the sample's GT list), ``labels``,
    ``label_weights``, ``bbox_targets``, ``dir_targets`` over the anchor table [N, 7] in
    (cell, size, rotation) order, and ``num_pos``."""
    C = cfg['num_classes']
    HW = anchors.shape[0] // (num_sizes * num_rots)
    per_size = anchors.view(HW, num_sizes, num_rots, 7)
    out = []
    for gb, gl in zip(gt_boxes, gt_labels):
        gl = gl.long()
        res = {k: [] for k in ('assigned', 'labels', 'label_weights', 'bbox_targets',
                               'dir_targets')}
        for s in range(num_sizes):
            a = per_size[:, s].reshape(-1, 7)
            sel = torch.nonzero(gl == s).reshape(-1) if cfg['assign_per_class'] else \
                torch.arange(len(gl), device=gl.device)
            N = a.shape[0]
            labels = torch.full((N,), C, dtype=torch.long, device=a.device)
            lw = a.new_zeros(N)
            bt = torch.zeros_like(a)
            dt = torch.zeros(N, dtype=torch.long, device=a.device)
            assigned = torch.zeros(N, dtype=torch.long, device=a.device)
            if len(sel) > 0:
                ov = bbox_overlaps(nearest_bev(gb[sel]), nearest_bev(a))
                asg = max_iou_assign(ov, *cfg['thr'][s])
                pos = torch.nonzero(asg > 0).reshape(-1)
                neg = torch.nonzero(asg == 0).reshape(-1)
                assigned = torch.where(asg > 0, sel[(asg - 1).clamp(min=0)] + 1, asg)
                if len(pos):
                    g = sel[asg[pos] - 1]
                    t = encode(a[pos], gb[g])
                    bt[pos] = t
                    dt[pos] = direction_target(a[pos], t, cfg['dir_offset'],
                                               cfg['dir_limit_offset'])
                    labels[pos] = gl[g]
                    lw[pos] = 1.0 if cfg.get('pos_weight', -1) <= 0 else cfg['pos_weight']
                lw[neg] = 1.0
            else:
                lw[:] = 1.0
            for k, v in (('assigned', assigned), ('labels', labels), ('label_weights', lw),
                         ('bbox_targets', bt), ('dir_targets', dt)):
                res[k].append(v.reshape(HW, 1, num_rots, *v.shape[1:]))
        res = {k: torch.cat(v, dim=1).reshape(HW * num_sizes * num_rots, *v[0].shape[3:])
               for k, v in res.items()}
        res['num_pos'] = int(((res['labels'] >= 0) & (res['labels'] < C)).sum())
        out.append(res)
    return out


class _FocalFn(torch.autograd.Function):
    """mmcv sigmoid_focal_loss (reduction 'none', no class weight): forward and backward as its
    CUDA kernels compute them, in the input's dtype."""

    @staticmethod
    def forward(ctx, x, t, gamma, alpha):
        p = torch.sigmoid(x)
        c = torch.arange(x.shape[1], device=x.device)[None]
        is_t = t[:, None] == c
        lp = torch.log(torch.clamp(p, min=FLT_MIN))
        lq = torch.log(torch.clamp(1 - p, min=FLT_MIN))
        loss = torch.where(is_t, -alpha * (1 - p)**gamma * lp, -(1 - alpha) * p**gamma * lq)
        ctx.save_for_backward(x, t)
        ctx.gamma, ctx.alpha = gamma, alpha
        return loss

    @staticmethod
    def backward(ctx, g):
        x, t = ctx.saved_tensors
        gamma, alpha = ctx.gamma, ctx.alpha
        p = torch.sigmoid(x)
        c = torch.arange(x.shape[1], device=x.device)[None]
        is_t = t[:, None] == c
        lp = torch.log(torch.clamp(p, min=FLT_MIN))
        lq = torch.log(torch.clamp(1 - p, min=FLT_MIN))
        gi = torch.where(is_t, -alpha * (1 - p)**gamma * (1 - p - gamma * p * lp),
                         -(1 - alpha) * p**gamma * (gamma * (1 - p) * lq - p))
        return gi * g, None, None, None


def sigmoid_focal_loss(x, t, gamma=2.0, alpha=0.25):
    return _FocalFn.apply(x, t, gamma, alpha)


def box2corners(b):
    """[P, 5] (x, y, w, h, yaw) -> [P, 4, 2], counter-clockwise (mmcv box2corners)."""
    x4 = b.new_tensor([0.5, -0.5, -0.5, 0.5]) * b[:, 2:3]
    y4 = b.new_tensor([0.5, 0.5, -0.5, -0.5]) * b[:, 3:4]
    c, s = torch.cos(b[:, 4:5]), torch.sin(b[:, 4:5])
    return torch.stack([x4 * c - y4 * s + b[:, 0:1], x4 * s + y4 * c + b[:, 1:2]], dim=-1)


def _in_box(p, q):
    a, bb, d = q[:, 0:1], q[:, 1:2], q[:, 3:4]
    ab, am, ad = bb - a, p - a, d - a
    pab = (ab * am).sum(-1) / (ab * ab).sum(-1)
    pad = (ad * am).sum(-1) / (ad * ad).sum(-1)
    return (pab > -1e-6) & (pab < 1 + 1e-6) & (pad > -1e-6) & (pad < 1 + 1e-6)


def oriented_box_intersection_2d(c1, c2):
    l1 = torch.cat([c1, c1[:, [1, 2, 3, 0]]], dim=-1)[:, :, None]    # P, 4, 1, 4
    l2 = torch.cat([c2, c2[:, [1, 2, 3, 0]]], dim=-1)[:, None]       # P, 1, 4, 4
    x1, y1, x2, y2 = l1.unbind(-1)
    x3, y3, x4, y4 = l2.unbind(-1)
    num = (x1 - x2) * (y3 - y4) - (y1 - y2) * (x3 - x4)
    den_t = (x1 - x3) * (y3 - y4) - (y1 - y3) * (x3 - x4)
    den_u = (x1 - x2) * (y1 - y3) - (y1 - y2) * (x1 - x3)
    zero = num == 0
    safe = torch.where(zero, torch.ones_like(num), num)
    t = torch.where(zero, -torch.ones_like(num), den_t / safe)
    u = torch.where(zero, -torch.ones_like(num), -den_u / safe)
    mask = (t > 0) & (t < 1) & (u > 0) & (u < 1)
    t = den_t / (num + 1e-8)
    inter = torch.stack([x1 + t * (x2 - x1), y1 + t * (y2 - y1)], dim=-1)
    P = c1.shape[0]
    verts = torch.cat([c1, c2, inter.reshape(P, 16, 2)], dim=1)       # P, 24, 2
    valid = torch.cat([_in_box(c1, c2), _in_box(c2, c1), mask.reshape(P, 16)], dim=1)
    verts = verts * valid[..., None].to(verts.dtype)
    n = valid.sum(1)
    mean = verts.sum(1) / n.clamp(min=1)[:, None].to(verts.dtype)
    rel = (verts - mean[:, None]).detach()
    ang = torch.atan2(rel[..., 1], rel[..., 0])
    ang = torch.where(valid, ang, torch.full_like(ang, 1e9))
    order = torch.argsort(ang, dim=1, stable=True)
    v = torch.gather(verts, 1, order[..., None].expand(-1, -1, 2))
    i = torch.arange(24, device=v.device)[None]
    nxt = torch.where(i + 1 < n[:, None], i + 1, torch.zeros_like(i))
    vn = torch.gather(v, 1, nxt[..., None].expand(-1, -1, 2))
    term = v[..., 0] * vn[..., 1] - v[..., 1] * vn[..., 0]
    term = torch.where(i < n[:, None], term, torch.zeros_like(term))
    area = term.sum(1).abs() / 2
    return torch.where(n >= 3, area, torch.zeros_like(area))


def diff_iou_rotated_3d(b1, b2):
    """[P, 7] x [P, 7] -> [P] (mmcv diff_iou_rotated_3d, unbatched)."""
    inter2 = oriented_box_intersection_2d(box2corners(b1[:, [0, 1, 3, 4, 6]]),
                                          box2corners(b2[:, [0, 1, 3, 4, 6]]))
    zmax1, zmin1 = b1[:, 2] + b1[:, 5] * 0.5, b1[:, 2] - b1[:, 5] * 0.5
    zmax2, zmin2 = b2[:, 2] + b2[:, 5] * 0.5, b2[:, 2] - b2[:, 5] * 0.5
    zo = (torch.min(zmax1, zmax2) - torch.max(zmin1, zmin2)).clamp(min=0.)
    inter = inter2 * zo
    v1 = b1[:, 3] * b1[:, 4] * b1[:, 5]
    v2 = b2[:, 3] * b2[:, 4] * b2[:, 5]
    return inter / (v1 + v2 - inter)


def dist_reduce_mean(t):
    """Mean over ranks under torch.distributed, else ``t``."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        t = t / dist.get_world_size()
        dist.all_reduce(t)
    return t


def smooth_l1_terms(pb, pt, cfg):
    """[P, 7] SmoothL1 terms of the positives' predictions ``pb`` against their targets ``pt``
    (``add_sin_difference``, then mmdet's smooth_l1_loss before its reduction)."""
    if cfg['diff_rad_by_sin']:
        pe = torch.sin(pb[:, 6:7]) * torch.cos(pt[:, 6:7])
        te = torch.cos(pb[:, 6:7]) * torch.sin(pt[:, 6:7])
        pb = torch.cat([pb[:, :6], pe], dim=-1)
        pt = torch.cat([pt[:, :6], te], dim=-1)
    diff = torch.abs(pb - pt)
    beta = cfg['beta']
    return torch.where(diff < beta, 0.5 * diff * diff / beta, diff - 0.5 * beta)


def losses(cls_score, bbox_pred, dir_pred, tg, anchors, cfg):
    """Loss dict of ``Anchor3DHead.loss`` (``cfg['liga']`` False) or of LIGA's ``loss_single``
    from per-sample targets ``tg``; the head outputs' dtype sets the arithmetic.  LIGA's IoU term
    uses each positive's own anchor and gives 0 without positives."""
    dt = cls_score.dtype
    B, _, ny, nx = cls_score.shape
    C = cfg['num_classes']
    labels = torch.cat([t['labels'] for t in tg])
    lw = torch.cat([t['label_weights'] for t in tg]).to(dt)
    btg = torch.cat([t['bbox_targets'] for t in tg]).to(dt)
    dtg = torch.cat([t['dir_targets'] for t in tg])
    n_total = sum(max(t['num_pos'], 1) for t in tg)
    if cfg['liga']:
        avg = dist_reduce_mean(cls_score.new_tensor(float(n_total)))
        den_cls = (avg + cfg['normalizer_clamp_value']) + FLT_EPS
        den = torch.clamp(avg, min=cfg['normalizer_clamp_value']) + FLT_EPS
    else:
        den_cls = den = n_total + FLT_EPS
    w = cfg['loss_weight']
    cls = cls_score.permute(0, 2, 3, 1).reshape(-1, C)
    # every term as mmdet forms it: loss * weight, sum / (avg_factor + eps), then loss_weight *
    l_cls = w[0] * ((sigmoid_focal_loss(cls, labels, cfg['gamma'], cfg['alpha']) *
                     lw[:, None]).sum() / den_cls)
    box = bbox_pred.permute(0, 2, 3, 1).reshape(-1, 7)
    pos = torch.nonzero((labels >= 0) & (labels < C)).reshape(-1)
    sl1 = smooth_l1_terms(box[pos], btg[pos], cfg)
    l_bbox = w[1] * ((sl1 * torch.ones_like(sl1)).sum() / den)
    d = dir_pred.permute(0, 2, 3, 1).reshape(-1, 2)[pos]
    ce = torch.nn.functional.cross_entropy(d, dtg[pos], reduction='none')
    l_dir = w[2] * ((ce * torch.ones_like(ce)).sum() / den)
    out = dict(loss_cls=l_cls, loss_bbox=l_bbox, loss_dir=l_dir)
    if cfg['with_iou']:
        an = anchors.to(dt).repeat(B, 1)[pos]
        if len(pos):
            bp = decode(an, box[pos])
            bt = decode(an, btg[pos])
            bt = torch.where(torch.isnan(bt), bp, bt)
            out['loss_iou'] = w[3] * ((1 - diff_iou_rotated_3d(bp, bt)).sum() / den)
        else:
            out['loss_iou'] = box.sum() * 0
    return out
