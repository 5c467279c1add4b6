"""Torch restatement of DfM's LiDAR imitation loss (``DfM.imitation_loss`` /
``get_imitation_reg_layer_loss``, detectors/dfm.py:455-539, with imitation_utils.py's
``NormalizeLayer('cw_scale')`` and ``WeightedL2WithSigmaLoss``), generalised as
``modules.DfMImitation`` is: any batch size with ragged per-sample GT, each sample tested against
its own boxes, the normaliser counting the whole batch and the loss divided by B.  At B = 1 it is
the reference.

The in-box mask and the positive counts are exact (the fp32 box test below, the same fp32 anchor
centres); the loss, gradients and scale run in the dtype of the inputs, so an fp64 call is the
reference up to the fp32 rounding of the dense conv and the mean over channels (a few ulp of
fp32).  ``pack`` / ``unpack`` state the one all-reduce the CUDA path performs: per pair
(count / world, count, sum_rows |t_c|), which gives the reference's dist_reduce_mean of the count
and its update's summed count and sums bit for bit.
"""
import torch

from depth_from_motion_b200 import modules


def anchor_centres(anchor_generator, ny, nx, device='cpu'):
    """(x per column [nx], y per row [ny]) of the BEV cells' anchor centres, fp32."""
    a = modules.grid_anchors(anchor_generator, ny, nx, device)
    A = a.shape[0] // (ny * nx)
    return a[0:nx * A:A, 0].clone(), a[0::nx * A, 1].clone()


def points_in_boxes_part(px, py, boxes):
    """mmcv 1.x points_in_boxes_part for points (px, py, 0) and LiDAR boxes [M, 7] whose z is
    taken as 0, in fp32 with every product and sum rounded on its own: the index of the first box
    that contains each point, -1 for none.  px, py: fp32 tensors of one shape."""
    out = torch.full(px.shape, -1, dtype=torch.long, device=px.device)
    boxes = boxes.to(px.device, torch.float32)
    for m in range(boxes.shape[0] - 1, -1, -1):   # the first box wins
        cx, cy, dx, dy, dz, rz = (boxes[m, k] for k in (0, 1, 3, 4, 5, 6))
        cz = dz * 0.5
        if bool(torch.abs(0.0 - cz) > dz * 0.5):
            continue
        cosa, sina = torch.cos(-rz), torch.sin(-rz)
        sx, sy = px - cx, py - cy
        lx = sx * cosa + sy * (-sina)
        ly = sx * sina + sy * cosa
        hx, hy = dx * 0.5, dy * 0.5
        inside = (lx > -hx) & (lx < hx) & (ly > -hy) & (ly < hy)
        out[inside] = m
    return out


def inbox_mask(ax, ay, gt_bboxes):
    """bool [B, ny, nx]: the cells whose anchor centre lies in one of the sample's GT."""
    py, px = torch.meshgrid(ay, ax, indexing='ij')
    return torch.stack([points_in_boxes_part(px, py, g) >= 0 for g in gt_bboxes])


def _rows(f):
    """[B, C, *spatial] -> [B * prod(spatial), C], the reference's channels-last view."""
    return f.permute(0, *range(2, f.dim()), 1).reshape(-1, f.shape[1])


def positives(inbox, teacher):
    """bool [rows]: in-box cell (repeated over z for a volume) and any teacher channel != 0."""
    m = inbox if teacher.dim() == 4 else \
        inbox.unsqueeze(1).expand(-1, teacher.shape[2], -1, -1)
    return m.reshape(-1) & torch.any(_rows(teacher) != 0, dim=-1)


def keep_positives(teacher, inbox, k):
    """Zeroes (in place) every teacher row but the first ``k`` positive ones, so the pair has
    exactly ``k`` positives (the n = 10 / 11 update gate, the normaliser clamp)."""
    pos = positives(inbox, teacher)
    idx = torch.nonzero(pos).view(-1)
    assert idx.numel() >= k, (idx.numel(), k)
    keep = torch.zeros_like(pos)
    keep[idx[:k]] = True
    spatial = (teacher.shape[0], 1) + teacher.shape[2:]
    return teacher.masked_fill_(~keep.view(teacher.shape[:1] + teacher.shape[2:]).view(spatial),
                                0)


def pack(counts, abs_sums, world=1):
    """The buffer the CUDA path all-reduces: per pair (count / world, count, sum |t|)."""
    parts = []
    for n, s in zip(counts, abs_sums):
        n = torch.as_tensor(n, dtype=torch.float32).reshape(1)
        parts += [n / world, n, s.reshape(-1).to(torch.float32)]
    return torch.cat(parts)


def unpack(buf, channels):
    """Inverse of ``pack``: [(mean count, count, sum |t|)] per pair."""
    out, off = [], 0
    for c in channels:
        out.append((buf[off], buf[off + 1], buf[off + 2:off + 2 + c]))
        off += 2 + c
    return out


def update_scale(scale, n, abs_sum, momentum=0.99):
    """NormalizeLayer.update('cw_scale') from the counts and sums over ranks, fp32."""
    if not float(n) > 10:
        return scale.clone()
    new = abs_sum.reshape(scale.shape) / n
    return scale * momentum + new * (1 - momentum)


def imitation_loss(xs, ts, ws, bs, scales, inbox, loss_weights, clamp=10.0, training=True,
                   reduce=None):
    """The per-pair losses and the scales after the call.  xs / ts: stereo and teacher features
    [B, C, (nz,) ny, nx]; ws [C, C(, 1...)] / bs [C] the 1x1 convs; scales [1, C] fp32 (not
    modified); inbox bool [B, ny, nx].  The loss runs in the dtype of xs (autograd works through
    it).  ``reduce``, when given, all-reduces the packed buffer (sum) in place, as the CUDA path
    does under torch.distributed; ``world`` is then its ``world_size`` attribute."""
    B = xs[0].shape[0]
    pos = [positives(inbox, t) for t in ts]
    counts = [p.sum() for p in pos]
    sums = [torch.sum(_rows(t)[p].abs(), dim=0) for t, p in zip(ts, pos)]
    buf = pack(counts, sums, getattr(reduce, 'world_size', 1))
    if reduce is not None:
        reduce(buf)
    red = unpack(buf, [x.shape[1] for x in xs])
    losses, new_scales = [], []
    for x, t, w, b, s, p, lw, (mean, n, asum) in zip(xs, ts, ws, bs, scales, pos, loss_weights,
                                                     red):
        C = x.shape[1]
        weight = 1.0 / torch.clamp(mean, min=clamp)                    # fp32, as reg_weights
        pred = _rows(x)[p] @ w.reshape(C, C).t().to(x.dtype) + b.to(x.dtype)
        tgt = (_rows(t)[p] / s).to(x.dtype)                           # fp32, as NormalizeLayer
        tgt = torch.where(torch.isnan(tgt), pred, tgt)
        row = (0.5 * (pred - tgt) ** 2 * weight.to(x.dtype)).mean(-1)
        losses.append(row.sum() / B * lw)
        new_scales.append(update_scale(s, n, asum) if training else s.clone())
    return losses, new_scales, [int(c) for c in counts]
