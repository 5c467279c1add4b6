"""Torch restatement of the anchor heads' ``get_bboxes_single`` (mmdet3d
dense_heads/anchor3d_head.py:459-547 with core/post_processing/box3d_nms.py:8-128, 231-268),
the oracle ``dfm_box_post_*`` is checked against.

Every step runs the reference's tensor ops in the reference's order, on whatever device the
inputs live on, so on the CPU it reproduces ``tests/golden/box_post.npz`` bit for bit and on the
GPU it sees the same sigmoid / exp rounding as the CUDA kernels.  Where the reference leaves an
order open (ties of ``topk`` and of the unstable sorts) the restatement fixes it the way the
kernels do: score descending, then anchor index ascending; the final ``max_num`` cut keeps
class-major order among equal scores.

mmcv's ``nms_rotated`` is not in the reference tree.  ``rotated_iou`` restates it with an exact
fp64 polygon intersection under ``NMS_ROTATED_ROT_SIGN``: corners at
``centre + R(NMS_ROTATED_ROT_SIGN * theta) (+-w/2, +-h/2)``, i.e. vertex 0 at
``(x + s h/2 + c w/2, y + c h/2 - s w/2)`` (mmcv-full 1.6.0 box_iou_rotated_utils.hpp, its
``clockwise=True`` default; box3d_nms.py:264 passes no flag).  IoU = inter / (w1 h1 + w2 h2 -
inter), and a later box is suppressed when IoU > nms_thr.
"""
import numpy as np
import torch

NMS_ROTATED_ROT_SIGN = -1.0


def corners(boxes):
    """[..., 5] (x, y, w, h, r) -> [..., 4, 2] counter-clockwise corners (fp64)."""
    b = boxes.double()
    x, y, w, h, r = b.unbind(-1)
    c, s = torch.cos(r), NMS_ROTATED_ROT_SIGN * torch.sin(r)
    u = torch.tensor([0.5, -0.5, -0.5, 0.5], dtype=torch.float64, device=b.device)
    v = torch.tensor([0.5, 0.5, -0.5, -0.5], dtype=torch.float64, device=b.device)
    uu, vv = u * w[..., None], v * h[..., None]
    px = x[..., None] + c[..., None] * uu - s[..., None] * vv
    py = y[..., None] + s[..., None] * uu + c[..., None] * vv
    return torch.stack((px, py), -1)


def _clip_edges(P, Q, keep_on_line):
    """2 x signed area swept by the parts of P's edges inside Q (Green's theorem), batched over
    the leading dims.  An edge on one of Q's edge lines counts only with `keep_on_line` and the
    same direction, so a shared boundary is counted once and a touching one not at all."""
    acc = torch.zeros(P.shape[:-2], dtype=torch.float64, device=P.device)
    for e in range(4):
        p0, d = P[..., e, :], P[..., (e + 1) % 4, :] - P[..., e, :]
        t0 = torch.zeros_like(acc)
        t1 = torch.ones_like(acc)
        ok = torch.ones_like(acc, dtype=torch.bool)
        for k in range(4):
            q0 = Q[..., k, :]
            ed = Q[..., (k + 1) % 4, :] - q0
            den = ed[..., 0] * d[..., 1] - ed[..., 1] * d[..., 0]
            rel = p0 - q0
            num = ed[..., 0] * rel[..., 1] - ed[..., 1] * rel[..., 0]
            par = den == 0
            same = (ed * d).sum(-1) > 0
            ok &= ~(par & ((num < 0) | ((num == 0) & ~(same & keep_on_line))))
            t = torch.where(par, torch.zeros_like(num), -num / torch.where(par, 1.0, den))
            t0 = torch.where(~par & (den > 0), torch.maximum(t0, t), t0)
            t1 = torch.where(~par & (den < 0), torch.minimum(t1, t), t1)
        cr = p0[..., 0] * d[..., 1] - p0[..., 1] * d[..., 0]
        acc = acc + torch.where(ok & (t1 > t0), (t1 - t0) * cr, torch.zeros_like(acc))
    return acc


def rotated_iou(a, b):
    """fp64 IoU of rotated boxes a [..., 5] and b [..., 5] (broadcast), on coordinates shifted
    to each pair's mean centre."""
    a, b = torch.broadcast_tensors(a.double(), b.double())
    cx = (a[..., 0] + b[..., 0]) / 2
    cy = (a[..., 1] + b[..., 1]) / 2
    shift = torch.stack((cx, cy, torch.zeros_like(cx), torch.zeros_like(cx),
                         torch.zeros_like(cx)), -1)
    A, B = corners(a - shift), corners(b - shift)
    inter = 0.5 * (_clip_edges(A, B, True) + _clip_edges(B, A, False))
    area_a, area_b = a[..., 2] * a[..., 3], b[..., 2] * b[..., 3]
    inter = torch.minimum(inter.clamp(min=0), torch.minimum(area_a, area_b))
    union = area_a + area_b - inter
    return torch.where(union > 0, inter / torch.where(union > 0, union, 1.0),
                       torch.zeros_like(union))


def nms_rotated(boxes, thr):
    """Greedy NMS over boxes [n, 5] already in processing order -> kept positions."""
    n = boxes.shape[0]
    removed = np.zeros(n, dtype=bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        if i + 1 < n:
            iou = rotated_iou(boxes[i:i + 1], boxes[i + 1:])
            removed[i + 1:] |= (iou > thr).cpu().numpy()
    return keep


def _order(scores, anchors):
    """Positions sorted by score descending, then anchor index ascending."""
    by_anchor = torch.argsort(anchors, stable=True)
    by_score = torch.argsort(scores[by_anchor], descending=True, stable=True)
    return by_anchor[by_score]


def decode(anchors, deltas):
    """DeltaXYZWLHRBBoxCoder.decode, op for op."""
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


def nms_box(boxes):
    """[x, y, dx, dy, yaw] through xywhr2xyxyr and nms_bev's way back (fp32 round trip)."""
    bev = boxes[:, [0, 1, 3, 4, 6]]
    half_w, half_h = bev[:, 2] / 2, bev[:, 3] / 2
    x1, y1 = bev[:, 0] - half_w, bev[:, 1] - half_h
    x2, y2 = bev[:, 0] + half_w, bev[:, 1] + half_h
    return torch.stack(((x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1, bev[:, 4]), -1)


def get_bboxes_single(cls_score, bbox_pred, dir_cls_pred, anchors, cfg, num_classes,
                      use_sigmoid=True, dir_offset=0.0, dir_limit_offset=0.0):
    """One sample: cls_score [A * ncol, H, W], bbox_pred [A * 7, H, W], dir_cls_pred
    [A * 2, H, W], anchors [H * W * A, 7]; num_classes = foreground classes.  Returns a dict
    with boxes [K, 7], scores [K], labels [K] and the stages: topk (anchor indices or None),
    candidates[c] / keep[c] (anchor indices in processing / keep order)."""
    ncol = num_classes + (0 if use_sigmoid else 1)
    dir_label = dir_cls_pred.permute(1, 2, 0).reshape(-1, 2).max(dim=-1)[1]
    cls = cls_score.permute(1, 2, 0).reshape(-1, ncol)
    scores = cls.sigmoid() if use_sigmoid else cls.softmax(-1)
    deltas = bbox_pred.permute(1, 2, 0).reshape(-1, 7)
    n = scores.shape[0]
    idx = torch.arange(n, device=scores.device)
    nms_pre = cfg.get('nms_pre', -1)
    topk = None
    if nms_pre > 0 and n > nms_pre:
        max_scores = scores.max(dim=1)[0] if use_sigmoid else scores[:, :-1].max(dim=1)[0]
        topk = _order(max_scores, idx)[:nms_pre]
        idx, anchors, deltas = topk, anchors[topk], deltas[topk]
        scores, dir_label = scores[topk], dir_label[topk]
    boxes = decode(anchors, deltas)
    bev = nms_box(boxes)
    score_thr = cfg.get('score_thr', 0)
    out_b, out_s, out_l, out_d = [], [], [], []
    cands, keeps = [], []
    for c in range(num_classes):
        sel = torch.nonzero(scores[:, c] > score_thr).flatten()
        order = sel[_order(scores[sel, c], idx[sel])]
        keep = order[nms_rotated(bev[order], cfg['nms_thr'])] if len(order) else order
        cands.append(idx[order])
        keeps.append(idx[keep])
        out_b.append(boxes[keep])
        out_s.append(scores[keep, c])
        out_l.append(torch.full((len(keep),), c, dtype=torch.long, device=boxes.device))
        out_d.append(dir_label[keep])
    boxes, scores = torch.cat(out_b), torch.cat(out_s)
    labels, dirs = torch.cat(out_l), torch.cat(out_d)
    if boxes.shape[0] > cfg['max_num']:
        inds = torch.argsort(scores, descending=True, stable=True)[:cfg['max_num']]
        boxes, scores, labels, dirs = boxes[inds], scores[inds], labels[inds], dirs[inds]
    if boxes.shape[0] > 0:
        val = boxes[..., 6] - dir_offset
        dir_rot = val - torch.floor(val / np.pi + dir_limit_offset) * np.pi
        boxes[..., 6] = dir_rot + dir_offset + np.pi * dirs.to(boxes.dtype)
    return dict(boxes=boxes, scores=scores, labels=labels, topk=topk, candidates=cands,
                keep=keeps)
