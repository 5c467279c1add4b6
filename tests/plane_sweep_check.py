"""fp64 referee of the plane-sweep cost volume and the per-element bound its CUDA warp is held
to (test_plane_sweep.py, test_backbone_layers.py).

The warp (``warp_coord`` + ``bilinear_taps``, csrc/common.cuh) evaluates the closed form
``[a, b, c] = z * A [u, v, 1]^T + t`` in fp32 with A, t rounded from the fp64 matrix
``M = P4 * cur2prev * P4^-1`` of ``make_warp_geom``.  The referee is ``oracle.build_dfm_cost``
run with float64 as the default dtype on fp64 inputs, with its cur half replaced by the exact
stride-lattice subsample (the kernel's cur half; the reference's fp64 round trip lands within
1e-12 of it).

Per prev-half element (channel k, plane z, lattice point x, y) the GPU must satisfy

    |gpu - ref| <= Lx * (dx + REF_PX) + Ly * (dy + REF_PX) + EPS_V_ULPS * u * sum_i |w_i f_i|

* (dx, dy) = K_DELTA * (the unit coordinate bounds of ``sample_points``): one unit roundoff u
  per magnitude the fp32 evaluation order carries, i.e. |u| (before and after the flip),
  |z| (|A_r0| |u| + |A_r1| |v| + |A_r2|) + |t_r| per row, amplified by the division as
  (R_a + |pu| R_c) / |c|, then the flip back, scale and crop of the result.  K_DELTA is the
  constant measured by emulating ``warp_coord`` in fp32 (``emulate_warp_coord``), with margin.
* Lx, Ly: the largest horizontal / vertical difference between adjacent taps of channel k
  (zero outside the map) over the 3 x 3 taps around the fp64 sample point rounded to the
  nearest pixel.  Bilinear interpolation is Lipschitz with these constants inside that
  neighbourhood, which holds both sample points while dx, dy < 0.5.
* The last term covers the fp32 weights and the fma chain over the four taps.

``grid_sample(zeros, align_corners=True)`` is continuous in the sample point, so no element is
excluded.  Elements where the bound is not a bound -- fp32 cannot place the sample within
NEAR_PX (the fp64 depth c in the previous camera is nearly 0) or the fp64 coordinate is beyond
GUARD -- are "near-singular": the tests require both sides to be 0 there or count them.
"""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O

U32 = 2.0 ** -24
# Calibrated by test_plane_sweep.py::test_delta_calibration: the worst |fp32 - fp64| / unit
# bound over the emulated geometries is 1.55 (DESIGN.md section 1); K_DELTA keeps a factor
# of 2.5 over it.
K_DELTA = 4.0
EPS_V_ULPS = 4.0
NEAR_PX = 0.25
GUARD = 1e7
# absolute floor of (dx, dy): the referee's own fp64 pixel -> 3-D -> pixel round trip lands
# within about 1e-13 px of the exact point, which matters where the exact coordinate and every
# magnitude of its fp32 evaluation are ~0 (the lattice origin under the identity pose)
REF_PX = 1e-9


@contextlib.contextmanager
def float64_default():
    """torch's default dtype is float64 inside the block (linspace, the crop tensor and every
    factory call of the oracle then build fp64 tensors) and restored on exit."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


class Geom:
    """What ``dfm_geometry_t`` carries, in fp64, plus the two sample factors."""

    def __init__(self, cam2img, cur2prev, ori_shape, flip=False, crop=(0, 0), scale=1.0,
                 fsf=1, csf=4):
        self.cam2img = np.asarray(cam2img, dtype=np.float64)
        self.cur2prev = np.asarray(cur2prev, dtype=np.float64).reshape(4, 4)
        self.ori_shape = tuple(ori_shape[:2])
        self.flip = bool(flip)
        self.crop = tuple(crop)
        self.scale = float(scale)
        self.fsf, self.csf = int(fsf), int(csf)

    @classmethod
    def from_meta(cls, meta, fsf=1, csf=4):
        c2p = meta['cur2prevs']
        c2p = c2p.detach().cpu().numpy() if isinstance(c2p, torch.Tensor) else c2p
        sf = meta.get('scale_factor', [1.0])
        return cls(meta['ori_cam2img'], np.asarray(c2p).reshape(-1, 4, 4)[0], meta['ori_shape'],
                   meta.get('flip', False), meta['crop_offset'],
                   sf[0] if hasattr(sf, '__len__') else sf, fsf, csf)

    def meta(self):
        """The img_meta keys ``modules.geometry_from_meta`` reads."""
        return dict(ori_cam2img=self.cam2img.tolist(),
                    cur2prevs=torch.from_numpy(self.cur2prev[None].copy()),
                    ori_shape=self.ori_shape + (3,), flip=self.flip, crop_offset=list(self.crop),
                    scale_factor=[self.scale] * 4)

    def matrix(self):
        """(A [3, 3], t [3]) of M = P4 cur2prev P4^-1 in fp64, as make_warp_geom forms it."""
        p = np.eye(4)
        p[:self.cam2img.shape[0], :self.cam2img.shape[1]] = self.cam2img
        p[3] = (0, 0, 0, 1)
        t = self.cur2prev.copy()
        t[3] = (0, 0, 0, 1)
        m = p @ t @ np.linalg.inv(p)
        return m[:3, :3], m[:3, 3]


def out_size(h, w, csf):
    return round(h / csf), round(w / csf)


# ---------------------------------------------------------------------------------------------
# referee
# ---------------------------------------------------------------------------------------------
def oracle_volume(cur, prev, depths, g, fn=O.build_dfm_cost):
    """``fn`` (oracle.build_dfm_cost, or the reference's own) under a float64 default dtype on
    fp64 copies of the inputs, on the features' device."""
    dev = cur.device
    cam = torch.as_tensor(g.cam2img, dtype=torch.float64, device=dev)[None]
    c2p = torch.as_tensor(g.cur2prev, dtype=torch.float64, device=dev)[None]
    with float64_default():
        return fn(cur.double(), prev.double(), depths.to(dev, torch.float64), g.fsf, g.csf, cam,
                  c2p, g.ori_shape, g.flip, g.crop, g.scale)


def lattice(cur, csf, ho, wo):
    """The cur half: the stride-lattice subsample, the same on every plane [1, C, 1, ho, wo]."""
    return cur[:, :, ::csf, ::csf][:, :, :ho, :wo].unsqueeze(2)


def referee(cur, prev, depths, g):
    """The fp64 referee volume [1, 2C, D, ho, wo] (cur half exactly on the lattice)."""
    vol = oracle_volume(cur, prev, depths, g)
    c = cur.shape[1]
    vol[:, :c] = lattice(cur.double(), g.csf, *vol.shape[-2:])
    return vol


# ---------------------------------------------------------------------------------------------
# sample points and the coordinate bound
# ---------------------------------------------------------------------------------------------
# planted defects of the separation test: the coordinate chain done wrong in one place
DEFECTS = ('shift_x', 'shift_y', 'align_corners_false', 'crop_after_scale', 'flip_about_w_minus_1')


def sample_points(g, depths, ho, wo, device='cpu', defect=None, shift=2e-3):
    """fp64 sample points of the prev half and the unit coordinate bounds, all [D, ho, wo]:
    dict(fx, fy, c, dx1, dy1).  `defect` (one of DEFECTS but 'align_corners_false', which is a
    sampler defect) plants an error in the coordinate chain."""
    f64 = torch.float64
    A, t = (torch.as_tensor(a, dtype=f64, device=device) for a in g.matrix())
    s, (cx, cy), w0, fl = g.scale, (float(g.crop[0]), float(g.crop[1])), float(g.ori_shape[1]), \
        float(g.flip)
    lat = g.fsf * g.csf
    xs = torch.arange(wo, dtype=f64, device=device) * lat
    ys = torch.arange(ho, dtype=f64, device=device) * lat
    if defect == 'crop_after_scale':
        ue, v = (xs / s + cx)[None, None, :], (ys / s + cy)[None, :, None]
    else:
        ue, v = ((xs + cx) / s)[None, None, :], ((ys + cy) / s)[None, :, None]
    z = depths.to(device, f64)[:, None, None]
    wf = w0 - 1 if defect == 'flip_about_w_minus_1' else w0
    u = wf - ue if g.flip else ue
    mu = ue.abs() + fl * u.abs()
    q = [A[r, 0] * u + A[r, 1] * v + A[r, 2] for r in range(3)]
    qm = [A[r, 0].abs() * mu + A[r, 1].abs() * v.abs() + A[r, 2].abs() for r in range(3)]
    a, b, c = (z * q[r] + t[r] for r in range(3))
    ra, rb, rc = (z.abs() * qm[r] + t[r].abs() for r in range(3))
    pu, pv = a / c, b / c
    pf = wf - pu if g.flip else pu
    if defect == 'crop_after_scale':
        fx, fy = (pf - cx) * s / g.fsf, (pv - cy) * s / g.fsf
    else:
        fx, fy = (pf * s - cx) / g.fsf, (pv * s - cy) / g.fsf
    if defect == 'shift_x':
        fx = fx + shift
    if defect == 'shift_y':
        fy = fy + shift
    ac = c.abs()
    dx1 = U32 / g.fsf * (s * (ra + pu.abs() * rc) / ac + s * (pu.abs() + fl * pf.abs()) +
                         abs(cx) + g.fsf * fx.abs())
    dy1 = U32 / g.fsf * (s * (rb + pv.abs() * rc) / ac + s * pv.abs() + abs(cy) +
                         g.fsf * fy.abs())
    return dict(fx=fx, fy=fy, c=c, dx1=dx1, dy1=dy1)


def _fma32(a, b, c):
    # a * b of two fp32 values is exact in fp64; one rounding to fp64, then to fp32
    return (a.astype(np.float64) * b + c).astype(np.float32)


def emulate_warp_coord(g, depths, ho, wo, contract):
    """csrc/common.cuh warp_coord in numpy fp32, op for op, on the WarpGeom make_warp_geom
    builds.  contract=True also fuses the two mul-add pairs nvcc may contract into fmas
    ((x * lattice + crop) and (pu * scale - crop)).  Returns (fx, fy) [D, ho, wo] fp32."""
    f32 = np.float32
    A, t = g.matrix()
    A, t = A.astype(f32), t.astype(f32)
    scale, inv_scale = f32(g.scale), f32(1.0 / g.scale)
    cx, cy, w0 = f32(g.crop[0]), f32(g.crop[1]), f32(g.ori_shape[1])
    lat, inv_fsf = f32(g.fsf * g.csf), f32(1) / f32(g.fsf)
    x = np.arange(wo, dtype=f32)[None, None, :]
    y = np.arange(ho, dtype=f32)[None, :, None]
    z = np.asarray(depths, dtype=f32)[:, None, None]
    if contract:
        u = (_fma32(x, lat, cx) * inv_scale).astype(f32)
        v = (_fma32(y, lat, cy) * inv_scale).astype(f32)
    else:
        u = ((x * lat).astype(f32) + cx).astype(f32) * inv_scale
        v = ((y * lat).astype(f32) + cy).astype(f32) * inv_scale
    u, v = u.astype(f32), v.astype(f32)
    if g.flip:
        u = (w0 - u).astype(f32)
    q = [_fma32(A[r, 0], u, _fma32(A[r, 1], v, A[r, 2])) for r in range(3)]
    a, b, c = (_fma32(np.broadcast_to(z, (len(z),) + q[r].shape[1:]), q[r], t[r])
               for r in range(3))
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        pu, pv = (a / c).astype(f32), (b / c).astype(f32)
        if g.flip:
            pu = (w0 - pu).astype(f32)
        if contract:
            fx = (_fma32(pu, scale, -cx) * inv_fsf).astype(f32)
            fy = (_fma32(pv, scale, -cy) * inv_fsf).astype(f32)
        else:
            fx = (((pu * scale).astype(f32) - cx).astype(f32) * inv_fsf).astype(f32)
            fy = (((pv * scale).astype(f32) - cy).astype(f32) * inv_fsf).astype(f32)
    return fx, fy


# ---------------------------------------------------------------------------------------------
# per-element bound
# ---------------------------------------------------------------------------------------------
def _finite_clamped(v, lim):
    return torch.where(torch.isfinite(v), v, torch.full_like(v, lim)).clamp(-lim, lim)


def bilinear(feat, fx, fy, align_corners=True):
    """grid_sample(zeros) of feat [1, C, H, W] fp64 at feature pixels (fx, fy) [D, ho, wo]:
    [1, C, D, ho, wo].  Non-finite or far points are moved to a far point (value 0)."""
    h, w = feat.shape[-2:]
    gx = _finite_clamped(fx, 1e6) / (w - 1) * 2 - 1
    gy = _finite_clamped(fy, 1e6) / (h - 1) * 2 - 1
    grid = torch.stack([gx, gy], -1).reshape(1, 1, -1, 2)
    out = F.grid_sample(feat, grid, mode='bilinear', padding_mode='zeros',
                        align_corners=align_corners)
    return out.view(1, feat.shape[1], *fx.shape)


def lipschitz_maps(feat):
    """(Lx, Ly) [C, H + 4, W + 4] of feat [C, H, W]: index (ry + 2, rx + 2) holds the largest
    horizontal / vertical adjacent difference over the 3 x 3 taps around pixel (ry, rx), with
    zeros outside the map."""
    p = F.pad(feat, (3, 3, 3, 3))
    hd = (p[:, :, 1:] - p[:, :, :-1]).abs()
    vd = (p[:, 1:, :] - p[:, :-1, :]).abs()
    return (F.max_pool2d(hd[None], (3, 2), 1)[0], F.max_pool2d(vd[None], (2, 3), 1)[0])


def near_singular(pts, k_delta=K_DELTA):
    return ((pts['dx1'] + pts['dy1']) * k_delta >= NEAR_PX) | \
        ~(pts['fx'].abs() < GUARD) | ~(pts['fy'].abs() < GUARD)


def prev_bound(prev, pts, k_delta=K_DELTA, maps=None):
    """Per-element bound [1, C, D, ho, wo] of the prev half (near-singular elements: +inf)."""
    prev = prev.double()
    h, w = prev.shape[-2:]
    lx, ly = maps if maps is not None else lipschitz_maps(prev[0])
    rx = (torch.floor(_finite_clamped(pts['fx'], 1e6) + 0.5).clamp(-2, w + 1) + 2).long()
    ry = (torch.floor(_finite_clamped(pts['fy'], 1e6) + 0.5).clamp(-2, h + 1) + 2).long()
    idx = (ry * (w + 4) + rx).reshape(-1)
    c = prev.shape[1]
    gx = lx.reshape(c, -1)[:, idx].view(1, c, *pts['fx'].shape)
    gy = ly.reshape(c, -1)[:, idx].view(1, c, *pts['fx'].shape)
    sabs = bilinear(prev.abs(), pts['fx'], pts['fy'])
    b = gx * (k_delta * pts['dx1'] + REF_PX) + gy * (k_delta * pts['dy1'] + REF_PX) + \
        EPS_V_ULPS * U32 * sabs
    return torch.where(near_singular(pts, k_delta)[None, None], torch.full_like(b, math.inf), b)


def warp_input_bound(prev, ref_prev, pts, c_cur):
    """Bound on |loader value - referee| for every channel of the 2C-channel volume, usable
    as a conv input bound: 0 on the cur half (exact), prev_bound on the prev half, and at
    near-singular elements |ref| + max |prev| (the loader's value is a convex combination of
    at most four taps with weights summing to at most 1 + a few ulps)."""
    b = prev_bound(prev, pts)
    worst = ref_prev.abs() + float(prev.abs().max()) * (1 + 8 * U32)
    b = torch.where(torch.isinf(b), worst, b)
    return torch.cat([torch.zeros_like(b[:, :c_cur]), b], 1)


def ratio(err, bound):
    """err / bound element-wise, 0 where err == 0 (bound 0: out-of-map samples)."""
    return torch.where(err == 0, torch.zeros_like(err), err / bound)
