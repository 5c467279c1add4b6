"""The rotated BEV IoU that decides get_bboxes' NMS, against an exact referee at degenerate
geometry: parallel edges on one line, nested and touching boxes, near-parallel yaws, far
translations and unwrapped yaws.

The referee builds each box's corner offsets in fp64 under ``NMS_ROTATED_ROT_SIGN``, adds them
to the (fp32) centre exactly in ``fractions.Fraction``, clips one quadrilateral by the other's
four half-planes (Sutherland-Hodgman) in exact rational arithmetic and takes the shoelace area.
It shares no code with ``box_post_oracle.rotated_iou``.

CPU: the fp64 restatement ``box_post_oracle.rotated_iou`` against the referee on every family
to 1e-12; the GPU bound sits >= 100x below the errors of an fp32 edge-clipping (Green's theorem)
IoU on the collinear family.
GPU: ``dfm_op_rotated_iou`` (the kernel's own ``bp_rect`` / ``bp_iou``) against the referee
within the bound, and its decision ``IoU > thr`` at the NMS thresholds."""
import ctypes
import functools
import math
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi
from tests import box_post_oracle as BP

U32 = 2.0 ** -24
THRESHOLDS = (0.01, 0.05, 0.25, 0.5)   # 0.05: Waymo nms_thr, 0.25: KITTI nms_thr
PERTURB = (1e-7, 1e-6, 1e-5, 1e-4, 1e-3)
# Error budget of the fp32 kernel IoU, with M = max |pair-centred corner coordinate| and
# L = perimeter_a + perimeter_b (the bounding circles meet, so M <= 3/8 L):
#   a corner is off by <= 8 u M (sincosf within 2 ulp, two products, a difference, the
#   centring add); a clip's side values and cut point move the boundary by <= 2 x that, so the
#   clipped area is off by <= 16 u M x perimeter(intersection) <= 8 u M L; the fan shoelace
#   (<= 6 triangles of |cross| <= 4 M^2, 3 roundings each, plus the sum) adds <= 72 u M^2
#   <= 27 u M L; IoU = I / (A + B - I) moves by <= 2 dI / max(A, B) + 4 u.
# 2 x (8 + 27) = 70, plus the 4 u, rounded up to the next power of two:
K_IOU = 128
SEPARATION = 100.0


def _axes(yaw):
    """Unit vectors of a box's w and h axes under the corner convention."""
    c, s = math.cos(yaw), BP.NMS_ROTATED_ROT_SIGN * math.sin(yaw)
    return (c, s), (-s, c)


def _at(yaw, du, dv):
    (ux, uy), (vx, vy) = _axes(yaw)
    return du * ux + dv * vx, du * uy + dv * vy


def _closed_form(rng):
    """Rows (family, a, b, closed-form IoU) with a, b = (x, y, w, h, yaw) before fp32
    rounding."""
    rows = []
    yaws = [0.0, math.pi / 2, math.pi / 4, math.pi] + list(rng.uniform(-math.pi, math.pi, 2))
    for yaw in yaws:
        for axis in (0, 1):                      # shifted along the w axis / the h axis
            for _ in range(4):
                w, h = rng.uniform(0.5, 5.0, 2)
                side = (w, h)[axis]
                s = rng.uniform(0.02, 0.98) * side
                x, y = _at(yaw, s, 0.0) if axis == 0 else _at(yaw, 0.0, s)
                rows.append(('shift_' + 'wh'[axis], (0.0, 0.0, w, h, yaw), (x, y, w, h, yaw),
                             (side - s) / (side + s)))
        w, h = rng.uniform(0.5, 5.0, 2)
        rows.append(('identical', (0.3, -0.2, w, h, yaw), (0.3, -0.2, w, h, yaw), 1.0))
        for lines in (1, 2):                     # nested, sharing one or two edge lines
            for _ in range(2):
                w, h = rng.uniform(1.0, 5.0, 2)
                f, g = rng.uniform(0.3, 0.9, 2)
                dv = (h - g * h) / 2 * (1.0 if lines == 2 else rng.uniform(-0.9, 0.9))
                x, y = _at(yaw, (w - f * w) / 2, dv)
                rows.append((f'nested_{lines}', (0.0, 0.0, w, h, yaw),
                             (x, y, f * w, g * h, yaw), f * g))
        for corner in (False, True):             # touching from outside
            for _ in range(2):
                w, h, w2, h2 = rng.uniform(0.5, 5.0, 4)
                dv = (h + h2) / 2 if corner else rng.uniform(-0.9, 0.9) * (h + h2) / 2
                x, y = _at(yaw, (w + w2) / 2, dv)
                rows.append(('touch_' + ('corner' if corner else 'edge'),
                             (0.0, 0.0, w, h, yaw), (x, y, w2, h2, yaw), 0.0))
        side = rng.uniform(1.0, 5.0)
        for f in (1 / math.sqrt(2), 0.5):        # 45-degree square in a square
            rows.append(('square45', (0.0, 0.0, side, side, yaw),
                         (0.0, 0.0, f * side, f * side, yaw + math.pi / 4), f * f))
        w = rng.uniform(2.0, 5.0)
        h = rng.uniform(0.3, 0.9) * w            # perpendicular cross
        rows.append(('cross', (0.0, 0.0, w, h, yaw), (0.0, 0.0, w, h, yaw + math.pi / 2),
                     h * h / (2 * w * h - h * h)))
    return rows


def _general(rng, n=300):
    """Random sizes and yaws, centres up to 1.1 x the sum of the circumradii apart (both sides
    of the bounding-circle early-out)."""
    rows = []
    for _ in range(n):
        w1, h1, w2, h2 = rng.uniform(0.2, 6.0, 4)
        r = (math.hypot(w1, h1) + math.hypot(w2, h2)) / 2
        d, phi = rng.uniform(0.0, 1.1) * r, rng.uniform(-math.pi, math.pi)
        rows.append(('general', (0.0, 0.0, w1, h1, rng.uniform(-math.pi, math.pi)),
                     (d * math.cos(phi), d * math.sin(phi), w2, h2,
                      rng.uniform(-math.pi, math.pi)), None))
    return rows


@functools.lru_cache(maxsize=None)
def cases():
    """(families [n], a [n, 5] fp32, b [n, 5] fp32, closed form [n] (nan where none)): every
    family as built, its b yaw perturbed by each of PERTURB, translated to |x|, |y| <= 80 m, and
    with yaws unwrapped by up to +-2 turns."""
    rng = np.random.RandomState(20261016)
    closed = _closed_form(rng)
    rows = list(closed)
    for d in PERTURB:
        rows += [(f'{f}_d{d:.0e}', a, b[:4] + (b[4] + d,), None) for f, a, b, _ in closed]
    rows += _general(rng)
    base = list(rows)
    for f, a, b, c in base:
        tx, ty = rng.uniform(-80.0, 80.0, 2)
        rows.append((f + '_far', (a[0] + tx, a[1] + ty) + a[2:], (b[0] + tx, b[1] + ty) + b[2:], c))
    for f, a, b, c in closed + base[-300:]:
        ka, kb = rng.randint(-2, 3, 2)
        rows.append((f + '_wrap', a[:4] + (a[4] + 2 * math.pi * ka,),
                     b[:4] + (b[4] + 2 * math.pi * kb,), c))
    fam = [r[0] for r in rows]
    a = np.array([r[1] for r in rows], dtype=np.float32)
    b = np.array([r[2] for r in rows], dtype=np.float32)
    cf = np.array([np.nan if r[3] is None else r[3] for r in rows])
    return fam, a, b, cf


# ------------------------------------------------------------------------ exact referee

def _corners_exact(box):
    x, y, w, h, r = (float(v) for v in box)
    c, s = math.cos(r), BP.NMS_ROTATED_ROT_SIGN * math.sin(r)
    out = []
    for u, v in ((0.5, 0.5), (-0.5, 0.5), (-0.5, -0.5), (0.5, -0.5)):
        uw, vh = u * w, v * h
        out.append((Fraction(x) + Fraction(c * uw - s * vh), Fraction(y) + Fraction(s * uw + c * vh)))
    return out


def _clip_exact(poly, q0, q1):
    ex, ey = q1[0] - q0[0], q1[1] - q0[1]
    side = [ex * (p[1] - q0[1]) - ey * (p[0] - q0[0]) for p in poly]
    out = []
    for i, p in enumerate(poly):
        j = (i + 1) % len(poly)
        if side[i] >= 0:
            out.append(p)
        if (side[i] >= 0) != (side[j] >= 0):
            t = side[i] / (side[i] - side[j])
            out.append((p[0] + t * (poly[j][0] - p[0]), p[1] + t * (poly[j][1] - p[1])))
    return out


def _area_exact(poly):
    return sum((p[0] * q[1] - p[1] * q[0] for p, q in zip(poly, poly[1:] + poly[:1])),
               Fraction(0)) / 2


def exact_iou(a, b):
    P, Q = _corners_exact(a), _corners_exact(b)
    poly = P
    for k in range(4):
        if not poly:
            break
        poly = _clip_exact(poly, Q[k], Q[(k + 1) % 4])
    inter = _area_exact(poly) if len(poly) >= 3 else Fraction(0)
    return float(inter / (_area_exact(P) + _area_exact(Q) - inter))


@functools.lru_cache(maxsize=None)
def exact():
    _, a, b, _ = cases()
    return np.array([exact_iou(x, y) for x, y in zip(a, b)])


def bound(a, b):
    """K_IOU u M (perimeter_a + perimeter_b) / min(area_a, area_b) per pair (fp64)."""
    a, b = a.astype(np.float64), b.astype(np.float64)
    cx, cy = (a[:, 0] + b[:, 0]) / 2, (a[:, 1] + b[:, 1]) / 2
    m = np.zeros(len(a))
    for box in (a, b):
        c, s = np.cos(box[:, 4]), BP.NMS_ROTATED_ROT_SIGN * np.sin(box[:, 4])
        for u, v in ((0.5, 0.5), (-0.5, 0.5), (-0.5, -0.5), (0.5, -0.5)):
            uw, vh = u * box[:, 2], v * box[:, 3]
            m = np.maximum(m, np.abs(box[:, 0] - cx + c * uw - s * vh))
            m = np.maximum(m, np.abs(box[:, 1] - cy + s * uw + c * vh))
    per = 2 * (a[:, 2] + a[:, 3] + b[:, 2] + b[:, 3])
    return K_IOU * U32 * m * per / np.minimum(a[:, 2] * a[:, 3], b[:, 2] * b[:, 3])


def _collinear(fam):
    return np.array([f.startswith('shift_') and '_d' not in f for f in fam])


# ---------------------------------------------------------------------------------- CPU

def test_case_families_cover_the_issue_list():
    fam, a, b, _ = cases()
    roots = {f.split('_d')[0].replace('_far', '').replace('_wrap', '') for f in fam}
    assert roots == {'shift_w', 'shift_h', 'identical', 'nested_1', 'nested_2', 'touch_edge',
                     'touch_corner', 'square45', 'cross', 'general'}
    assert np.abs(np.concatenate((a[:, :2], b[:, :2]))).max() > 70.0
    assert np.abs(np.concatenate((a[:, 4], b[:, 4]))).max() > 3 * math.pi
    g = np.array([f.startswith('general') for f in fam])
    d = np.hypot(a[g, 0] - b[g, 0], a[g, 1] - b[g, 1])
    rr = (np.hypot(a[g, 2], a[g, 3]) + np.hypot(b[g, 2], b[g, 3])) / 2
    assert (d > rr).sum() > 10 and (d < rr).sum() > 100     # both sides of the early-out


def test_referee_matches_closed_forms():
    """The closed forms hold for the unrounded boxes; fp32 rounding of centres, sizes and yaws
    moves the exact IoU by a few 1e-7 relative to the box scale."""
    fam, a, b, cf = cases()
    ex = exact()
    sel = ~np.isnan(cf)
    err = np.abs(ex[sel] - cf[sel])
    tol = 1e-5 + 16 * U32 * (1 + np.abs(a[sel, :2]).max(1)) * 8 / np.minimum(
        a[sel, 2] * a[sel, 3], b[sel, 2] * b[sel, 3])
    assert bool((err <= tol).all()), (float(err.max()), np.array(fam)[sel][np.argmax(err - tol)])
    assert float(np.abs(ex[np.array([f == 'identical' for f in fam])] - 1).max()) < 1e-6


def test_restatement_matches_exact_referee():
    fam, a, b, _ = cases()
    with torch.no_grad():
        got = BP.rotated_iou(torch.from_numpy(a), torch.from_numpy(b)).numpy()
    err = np.abs(got - exact())
    worst = int(np.argmax(err))
    assert float(err.max()) <= 1e-12, (fam[worst], a[worst], b[worst], float(err.max()))


# An fp32 IoU that clips each rectangle's edges to the other and sums the swept area by Green's
# theorem (each polygon's edges clipped independently, an edge taken as parallel only when the
# cross product is exactly 0): the form this kernel replaced.  Host C++ with the kernel's
# operation order and no contraction; libm sinf / cosf stand in for the device sincosf.
_GREEN_SRC = r'''
#include <math.h>
static float cr(float ax, float ay, float bx, float by) { return ax * by - ay * bx; }
struct R { float x, y, area, radius, ox[4], oy[4]; };
static R rect(const float* bv) {
  R r; r.x = bv[0]; r.y = bv[1];
  const float w = bv[2], h = bv[3];
  r.area = w * h; r.radius = 0.5f * sqrtf(w * w + h * h);
  float sn = -sinf(bv[4]), cs = cosf(bv[4]);
  const float us[4] = {0.5f, -0.5f, -0.5f, 0.5f}, vs[4] = {0.5f, 0.5f, -0.5f, -0.5f};
  for (int k = 0; k < 4; ++k) {
    const float u = us[k] * w, v = vs[k] * h;
    r.ox[k] = cs * u - sn * v; r.oy[k] = sn * u + cs * v;
  }
  return r;
}
static float clip_edges(const float* px, const float* py, const float* qx, const float* qy,
                        bool keep_on_line) {
  float acc = 0.f;
  for (int e = 0; e < 4; ++e) {
    const float x0 = px[e], y0 = py[e];
    const float dx = px[(e + 1) & 3] - x0, dy = py[(e + 1) & 3] - y0;
    float t0 = 0.f, t1 = 1.f; bool ok = true;
    for (int k = 0; k < 4; ++k) {
      const float ex = qx[(k + 1) & 3] - qx[k], ey = qy[(k + 1) & 3] - qy[k];
      const float den = cr(ex, ey, dx, dy), num = cr(ex, ey, x0 - qx[k], y0 - qy[k]);
      if (den == 0.f) {
        if (num < 0.f || (num == 0.f && !(keep_on_line && ex * dx + ey * dy > 0.f))) ok = false;
      } else {
        const float t = -num / den;
        if (den > 0.f) t0 = fmaxf(t0, t); else t1 = fminf(t1, t);
      }
    }
    if (ok && t1 > t0) acc += (t1 - t0) * cr(x0, y0, dx, dy);
  }
  return acc;
}
extern "C" void green_iou(const float* A, const float* B, int n, float* out) {
  for (int i = 0; i < n; ++i) {
    const R a = rect(A + 5 * i), b = rect(B + 5 * i);
    const float dx = b.x - a.x, dy = b.y - a.y, rr = a.radius + b.radius;
    if (dx * dx + dy * dy > rr * rr * 1.0001f + 1e-6f) { out[i] = 0.f; continue; }
    const float cx = (a.x + b.x) * 0.5f, cy = (a.y + b.y) * 0.5f;
    float pax[4], pay[4], pbx[4], pby[4];
    for (int k = 0; k < 4; ++k) {
      pax[k] = (a.x - cx) + a.ox[k]; pay[k] = (a.y - cy) + a.oy[k];
      pbx[k] = (b.x - cx) + b.ox[k]; pby[k] = (b.y - cy) + b.oy[k];
    }
    float inter = 0.5f * (clip_edges(pax, pay, pbx, pby, true) +
                          clip_edges(pbx, pby, pax, pay, false));
    inter = fminf(fmaxf(inter, 0.f), fminf(a.area, b.area));
    const float uni = a.area + b.area - inter;
    out[i] = uni > 0.f ? inter / uni : 0.f;
  }
}
'''


def green_iou(a, b, tmp_path):
    """The edge-clipping IoU above on fp32 [n, 5] pairs, built with g++ in tmp_path."""
    src, so = tmp_path / 'green.cpp', tmp_path / 'green.so'
    if not so.exists():
        src.write_text(_GREEN_SRC)
        subprocess.run(['g++', '-O2', '-ffp-contract=off', '-fno-fast-math', '-shared', '-fPIC',
                        '-o', str(so), str(src)], check=True)
    A = np.ascontiguousarray(a, dtype=np.float32)
    B = np.ascontiguousarray(b, dtype=np.float32)
    out = np.zeros(len(A), dtype=np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    ctypes.CDLL(str(so)).green_iou(A.ctypes.data_as(fp), B.ctypes.data_as(fp), len(A),
                                   out.ctypes.data_as(fp))
    return out.astype(np.float64)


@pytest.mark.skipif(shutil.which('g++') is None, reason='no C++ compiler')
def test_bound_separates_the_edge_clipping_iou(tmp_path):
    """On the collinear family (equal boxes shifted along one axis, at the origin and 80 m out),
    the edge-clipping IoU misses the exact IoU by >= SEPARATION x the bound on many pairs, so the
    GPU test's bound would catch it."""
    fam, a, b, _ = cases()
    sel = _collinear(fam)
    A, B = a[sel], b[sel]
    err = np.abs(green_iou(A, B, tmp_path) - exact()[sel])
    ratio = err / bound(A, B)
    print('collinear pairs', len(A), 'worst error', float(err.max()), 'worst error / bound',
          float(ratio.max()), 'pairs >= 100 x bound', int((ratio >= SEPARATION).sum()))
    assert float(ratio.max()) >= 10 * SEPARATION
    assert int((ratio >= SEPARATION).sum()) >= len(A) // 20


# ------------------------------------------------------------------ dense near-duplicates

@functools.lru_cache(maxsize=None)
def near_duplicates(n=40000):
    """3 n pairs of near-identical boxes at |x|, |y| <= 80 m, the pairs NMS must suppress:
    every field of b moved by -4..4 ulp from a's; b's yaw moved by 1e-8 .. 1e-6 either way; b
    the same rectangle at yaw + pi.  Their corners sit within rounding of several clip lines at
    once, where rounding adds vertices to the clipped polygon."""
    rng = np.random.RandomState(31)
    a = np.stack([rng.uniform(-80, 80, 3 * n), rng.uniform(-80, 80, 3 * n),
                  rng.uniform(0.5, 6.0, 3 * n), rng.uniform(0.5, 6.0, 3 * n),
                  rng.uniform(-math.pi, math.pi, 3 * n)], 1).astype(np.float32)
    b = a.copy()
    b[:n] = (a[:n].view(np.int32) + rng.randint(-4, 5, (n, 5)).astype(np.int32)).view(np.float32)
    d = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-8, -6, n)
    b[n:2 * n, 4] = (a[n:2 * n, 4].astype(np.float64) + d).astype(np.float32)
    b[2 * n:, 4] = (a[2 * n:, 4].astype(np.float64) + math.pi).astype(np.float32)
    return a, b


def test_restatement_on_near_duplicates_matches_exact_referee():
    """A seeded 1500-pair sample of the near-duplicate family (500 of each kind) through the
    exact referee; the GPU test compares the kernel with the restatement on all of it."""
    a, b = near_duplicates()
    n = len(a) // 3
    idx = np.concatenate([np.arange(k * n, k * n + 500) for k in range(3)])
    ex = np.array([exact_iou(a[i], b[i]) for i in idx])
    with torch.no_grad():
        got = BP.rotated_iou(torch.from_numpy(a[idx]), torch.from_numpy(b[idx])).numpy()
    assert float(np.abs(got - ex).max()) <= 1e-12
    assert float(ex.min()) > 0.99


def test_rotated_iou_entry_point_is_declared():
    assert 'dfm_op_rotated_iou' in capi.SYMBOLS


# ---------------------------------------------------------------------------------- GPU

def gpu_iou(a, b):
    """dfm_op_rotated_iou on fp32 [n, 5] numpy pairs."""
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    out = torch.full((len(a),), float('nan'), device='cuda')
    L = capi.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    capi.check(L.dfm_op_rotated_iou(p(da), p(db), len(a), p(out), None), 'dfm_op_rotated_iou')
    capi.sync_check()
    return out.cpu().double().numpy()


@pytest.mark.gpu
def test_entry_point_rejects_bad_arguments():
    L = capi.lib()
    t = torch.zeros(5, device='cuda')
    p = ctypes.c_void_p(t.data_ptr())
    assert L.dfm_op_rotated_iou(p, p, 0, p, None) == 1
    assert L.dfm_op_rotated_iou(p, p, -3, p, None) == 1
    assert L.dfm_op_rotated_iou(None, p, 1, p, None) == 1
    assert L.dfm_op_rotated_iou(p, None, 1, p, None) == 1
    assert L.dfm_op_rotated_iou(p, p, 1, None, None) == 1


@pytest.mark.gpu
def test_kernel_iou_within_bound_of_exact():
    fam, a, b, _ = cases()
    got, ex, bd = gpu_iou(a, b), exact(), bound(a, b)
    err = np.abs(got - ex)
    bad = np.nonzero(~(err <= bd))[0]
    fams = sorted({fam[i] for i in bad})
    col = _collinear(fam)
    print('pairs', len(a), 'worst error', float(err.max()), 'worst error / bound',
          float((err / bd).max()), 'collinear worst error', float(err[col].max()))
    assert len(bad) == 0, (len(bad), fams[:12], [(float(got[i]), float(ex[i]), float(bd[i]))
                                                 for i in bad[:5]])


@pytest.mark.gpu
def test_kernel_iou_on_near_duplicates():
    """120000 near-duplicate pairs: within the bound of the fp64 restatement (itself within
    1e-12 of exact on this family), and every one suppressed at each NMS threshold."""
    a, b = near_duplicates()
    got = gpu_iou(a, b)
    with torch.no_grad():
        ref = BP.rotated_iou(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()).cpu().numpy()
    err = np.abs(got - ref)
    bd = bound(a, b) + 1e-12
    print('near-duplicate pairs', len(a), 'worst error', float(err.max()), 'worst error / bound',
          float((err / bd).max()), 'lowest IoU', float(got.min()))
    bad = np.nonzero(~(err <= bd))[0]
    assert len(bad) == 0, (len(bad), [(a[i].tolist(), b[i].tolist(), float(got[i]),
                                       float(ref[i])) for i in bad[:3]])
    assert bool((got > max(THRESHOLDS)).all())


@pytest.mark.gpu
@pytest.mark.parametrize('thr', THRESHOLDS)
def test_kernel_nms_decision_matches_exact(thr):
    fam, a, b, _ = cases()
    got, ex, bd = gpu_iou(a, b), exact(), bound(a, b)
    clear = np.abs(ex - thr) > bd
    wrong = np.nonzero(clear & ((got > thr) != (ex > thr)))[0]
    assert clear.sum() > 0.9 * len(a)
    assert len(wrong) == 0, (len(wrong), sorted({fam[i] for i in wrong})[:12])
