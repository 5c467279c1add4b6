"""Torch restatement of ``DepthHead.loss`` (dense_heads/depth_head.py:75-188) for the ce /
balanced_ce / focal / balanced_focal types, and the inputs of the golden fixture
(tests/golden/make_depth_loss_golden.py writes it from the reference's own code).

``dense_loss`` takes the ``[B*N, fD, fH, fW]`` volume the reference call site passes and runs the
reference's operations in its order, so in fp32 on the CPU it reproduces the fixture bit for bit.
``column_loss`` takes the low-res ``[B, N, D, H, W]`` logits and builds only the masked
columns (the separable trilinear align_corners interpolation, in the input's dtype), so it runs at
the shipped training shape in fp64.  Both return ``loss_weight**2 * loss``: the reference
multiplies by its ``loss_weight`` and by a per-type weight that equals it."""
import numpy as np
import torch
import torch.nn.functional as F

from depth_from_motion_b200 import synthetic as syn
from oracle import dfm_oracle

TYPES = ('ce', 'balanced_ce', 'focal', 'balanced_focal')
# the shipped KITTI configs (configs/dfm/*kitti*.py: depth_head.depth_loss and depth_cfg)
SHIPPED_LOSS = dict(type='balanced_focal', loss_weight=1.0, fg_weight=5, bg_weight=1, alpha=1,
                    gamma=2)
MIN_DEPTH, MAX_DEPTH = 2, 59.6


def loss_config(loss_type, loss_weight=1.0):
    """A ``depth_loss`` dict of ``loss_type`` with the shipped constants."""
    cfg = dict(type=loss_type, loss_weight=loss_weight)
    if loss_type.startswith('balanced'):
        cfg.update(fg_weight=SHIPPED_LOSS['fg_weight'], bg_weight=SHIPPED_LOSS['bg_weight'])
    if loss_type.endswith('focal'):
        cfg.update(alpha=SHIPPED_LOSS['alpha'], gamma=SHIPPED_LOSS['gamma'])
    return cfg


def samples_for(num_planes, factor=4):
    """``DfM.prepare_depth``'s full-resolution bin centres for D = num_planes."""
    return dfm_oracle.depth_samples(syn.depth_cfg_for(num_planes, factor))


def _reduce(cost, gt, fgm, samples, cfg, depth_preds):
    """The loss of the masked columns ``cost`` [M, fD] with depths ``gt`` [M]."""
    t = cfg['type']
    if t not in TYPES:
        raise NotImplementedError(t)
    if gt.shape[0] == 0:
        return depth_preds.mean() * 0.0
    interval = samples[1] - samples[0]
    log_p = F.log_softmax(cost, dim=1)
    p = 1 - (torch.abs(samples - gt.unsqueeze(-1)) / interval).clamp(max=1.0)
    if t.endswith('focal'):
        per = -(p * (cfg['alpha'] * (1 - log_p.exp()).pow(cfg['gamma']) * log_p)).sum(-1)
    else:
        per = -(p * log_p).sum(-1)
    if t.startswith('balanced'):
        loss = (cfg['fg_weight'] * per[fgm]).sum() + (cfg['bg_weight'] * per[~fgm]).sum()
        loss = loss / len(gt)
    else:
        loss = per.mean()
    return cfg['loss_weight'] * cfg['loss_weight'] * loss


def _mask(depth_img, min_depth, max_depth):
    return (depth_img > min_depth) & (depth_img < max_depth)


def dense_loss(vol, depth_img, fgmask, samples, cfg, depth_preds, min_depth=MIN_DEPTH,
               max_depth=MAX_DEPTH):
    """Loss of the dense volume ``vol`` [B*N, fD, fH, fW]."""
    mask = _mask(depth_img, min_depth, max_depth)
    fgm = fgmask[mask].bool() if fgmask is not None else None
    cost = vol.permute(0, 2, 3, 1)[mask]
    return _reduce(cost, depth_img[mask].to(vol.dtype), fgm, samples.to(vol.dtype), cfg,
                   depth_preds)


def _taps(n_in, n_out, idx, dtype, wdtype):
    """ATen's align_corners source index of full-res ``idx`` computed in ``wdtype`` (ATen uses
    the input's dtype): the two taps and their weights, as ``dtype``.  The scale is a true
    division on the host, as ATen's (a CUDA tensor divided by a number is multiplied by the
    reciprocal instead)."""
    scale = torch.tensor(float(n_in - 1), dtype=wdtype) / (n_out - 1) if n_out > 1 else \
        torch.zeros((), dtype=wdtype)
    src = scale.to(idx.device) * idx.to(wdtype)
    i0 = torch.clamp(src.long(), max=n_in - 1)
    l1 = src - i0.to(wdtype)
    i1 = torch.clamp(i0 + 1, max=n_in - 1)
    return i0, i1, (1 - l1).to(dtype), l1.to(dtype)


def column_loss(cost, depth_img, fgmask, samples, cfg, depth_preds, factor=4,
                min_depth=MIN_DEPTH, max_depth=MAX_DEPTH, weights_dtype=None):
    """Loss of the x-factor trilinear upsampling of ``cost`` [B, N, D, H, W], built only under
    the masked pixels; differentiable with respect to ``cost``.  The interpolation weights are
    formed in ``weights_dtype`` (default: the cost's, as ``F.interpolate`` does).  An fp32
    upsampling's source indices carry absolute errors up to ulp(index) / 2 (~1e-5 at index 320),
    so an fp64 check of an fp32 path takes the fp32 weights and computes in fp64 from them."""
    b, nv, d, h, w = cost.shape
    c = cost.reshape(b * nv, d, h, w)
    dt = cost.dtype
    wd = weights_dtype or dt
    mask = _mask(depth_img, min_depth, max_depth)
    ni, yy, xx = mask.nonzero(as_tuple=True)
    y0, y1, wy0, wy1 = _taps(h, factor * h, yy, dt, wd)
    x0, x1, wx0, wx1 = _taps(w, factor * w, xx, dt, wd)

    def row(y):
        return wx0[:, None] * c[ni, :, y, x0] + wx1[:, None] * c[ni, :, y, x1]

    cols = wy0[:, None] * row(y0) + wy1[:, None] * row(y1)            # [M, D]
    k = torch.arange(factor * d, device=cost.device)
    z0, z1, l0, l1 = _taps(d, factor * d, k, dt, wd)
    vals = cols[:, z0] * l0 + cols[:, z1] * l1                          # [M, fD]
    fgm = fgmask[mask].bool() if fgmask is not None else None
    return _reduce(vals, depth_img[mask].to(dt), fgm, samples.to(cost.device, dt), cfg,
                   depth_preds)


# ---- the golden fixture's cases: name -> (loss type, loss_weight, depth-map variant, seed) ----
GOLDEN_SHAPE = dict(n=2, D=8, H=6, W=10, f=4)
GOLDEN_CASES = {
    'ce': ('ce', 1.0, 'sparse', 3),
    'balanced_ce': ('balanced_ce', 1.0, 'sparse', 4),
    'focal': ('focal', 1.0, 'sparse', 5),
    'balanced_focal': ('balanced_focal', 1.0, 'sparse', 6),
    'balanced_focal_weight2': ('balanced_focal', 2.0, 'sparse', 7),
    'edges_focal': ('focal', 1.0, 'edges', 8),
    'edges_balanced_ce': ('balanced_ce', 1.0, 'edges', 9),
    'no_masked_pixel': ('balanced_focal', 1.0, 'empty', 10),
}


def edge_depths(samples, min_depth=MIN_DEPTH, max_depth=MAX_DEPTH):
    """Depths at the mask bounds (fp32(min), fp32(max) and their nextafter inward and
    outward), exactly on bin centres and exactly halfway between two."""
    f32 = np.float32
    lo, hi = f32(min_depth), f32(max_depth)
    s = samples.numpy()
    mids = [(s[i] + s[i + 1]) / f32(2) for i in (0, 5, len(s) - 2)]
    vals = [lo, np.nextafter(lo, f32(np.inf)), np.nextafter(lo, f32(-np.inf)), hi,
            np.nextafter(hi, f32(-np.inf)), np.nextafter(hi, f32(np.inf)),
            s[0], s[1], s[7], s[len(s) // 2], s[-1], *mids]
    return np.array(vals, np.float32)


def golden_inputs(name):
    """(loss config, cost [n, 1, D, H, W], depth [n, fH, fW], fgmask int32, depth_preds,
    samples) of golden case ``name``."""
    t, lw, variant, seed = GOLDEN_CASES[name]
    g = GOLDEN_SHAPE
    cost, depth, fg = syn.make_depth_loss_case(seed, g['n'], g['D'], g['H'], g['W'], g['f'],
                                               density=0.3)
    samples = samples_for(g['D'], g['f'])
    if variant == 'edges':
        depth[0] = 0.0                      # image 0 has no masked pixel, image 1 has them
        e = torch.from_numpy(edge_depths(samples))
        depth[1, 3, 5:5 + len(e)] = e
    elif variant == 'empty':
        depth.zero_()
    preds = syn.smooth_field(np.random.RandomState(seed + 100), g['n'], g['f'] * g['H'],
                             g['f'] * g['W'])[0] * 10 + 30
    return loss_config(t, lw), cost, depth, fg, preds, samples
