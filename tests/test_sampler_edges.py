"""The voxel lift, the FrustumToVoxel gather and voxel_sample, bit for bit at exactly
representable image and depth edges.

The realistic-rig tests of these samplers (test_gpu_parity.py, test_stage_layers.py) excuse
every element whose sample point lies near a validity edge or a nearest-tap tie: the oracle
projects in fp32 through a BLAS matmul whose summation order is not the kernels', so near an
edge neither side's decision is the right one.  Here the geometry is built so that every fp32
operation of each projection is exact: power-of-two focal lengths, integer principal points,
axis-permutation rotations, dyadic translations and voxel centres, depths whose magnitudes are
0 or powers of two, scale factors of 1 or 0.5, integer crops, and feature / image sizes that
make the normalise-unnormalise chain a power-of-two scaling.  Every summation order then gives
the same bits, the reference's decision at an edge or a tie is unambiguous, and the kernels
must reproduce it with no tolerance and no excused elements.

CPU: each case is exact (fp32 in two summation orders and fp64 agree bit for bit), each case
holds the edges it exists for, a numpy restatement of each kernel's decisions equals the
oracle, and each planted defect of those decisions changes at least one output element.
GPU: the lift through all four entry points, the frustum gather on both softmax paths and
three constructor variants, and voxel_sample in both modes, against the fp64 oracle.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O

f32 = np.float32


def axis(lo, step, n):
    """n voxel centres lo, lo + step, ...: dyadic, so each one is exact in fp32."""
    return (np.arange(n) * step + lo).astype(f32)


def agree(*vals):
    """All arrays hold the same values bit for bit (NaN equal to NaN, signed infinities)."""
    a = np.asarray(vals[0], dtype=np.float64)
    return all(np.array_equal(a, np.asarray(v, dtype=np.float64), equal_nan=True)
               for v in vals[1:])


def project(m, p, prec, order):
    """Rows 0..2 of [p, 1] @ m.T in `prec`, every product and sum rounded, in one of two
    summation orders."""
    m = np.asarray(m, dtype=f32).astype(prec)
    x, y, z = (np.asarray(c, dtype=f32).astype(prec) for c in p)
    rows = []
    for r in range(3):
        t0, t1, t2 = x * m[r, 0], y * m[r, 1], z * m[r, 2]
        rows.append(((t0 + t1) + t2) + m[r, 3] if order == 0 else m[r, 3] + (t2 + (t1 + t0)))
    return rows


def round_nearest(x, away=False):
    """nearbyint (half to even, what grid_sample and the kernels use), or the planted
    half-away-from-zero rule."""
    with np.errstate(invalid='ignore'):
        return np.sign(x) * np.floor(np.abs(x) + 0.5) if away else np.rint(x)


def tie_splits(x):
    """Positions where half-even and half-away rounding pick different taps."""
    with np.errstate(invalid='ignore'):
        return np.isfinite(x) & (round_nearest(x) != round_nearest(x, away=True))


# ---------------------------------------------------------------------------------------------
# MultiViewDfM lift (lift_kernel / lift_voxel_kernel / lift_cl_kernel, csrc/simt_kernels.cuh)
# ---------------------------------------------------------------------------------------------
LIFT_IN_HW = (64, 128)
# (c / 128 * 2 - 1 + 1) / 2 * 32 = c / 4 and (c / 64 * 2 - 1 + 1) / 2 * 16 = c / 4: every tap
# coordinate is exact and ties land on .5 at c = 4k + 2
LIFT_FEAT_HW = (17, 33)
LIFT_N_VOXELS = [5, 81, 41]
LIFT_RANGE = [-2.5, -40.5, -20.5, 2.5, 40.5, 20.5]
LIFT_AXES = (axis(-2, 1, 5), axis(-40, 1, 81), axis(-20, 1, 41))
LIFT_IMG_W = 120     # img_shape[s][1] != input_w: the flip is about the unpadded width
LIFT_CASES = {
    'plain': dict(f=2., c=(64., 32.), scale=1., crop=(0., 0.)),
    'aug': dict(f=4., c=(128., 64.), scale=.5, crop=(2., 2.)),
}
# view 0 looks along +x, view 1 along -x (x_cam, y_cam, z_cam from lidar x, y, z); depth is
# +-x in {-2, ..., 2}: zero, negative and power-of-two depths in every view
LIFT_ROTATIONS = ([[0, -1, 0], [0, 0, -1], [1, 0, 0]], [[0, 1, 0], [0, 0, -1], [-1, 0, 0]])


def lift_case(name, t, flip):
    a = LIFT_CASES[name]
    k = np.array([[a['f'], 0, a['c'][0], 0], [0, a['f'], a['c'][1], 0], [0, 0, 1, 0],
                  [0, 0, 0, 1]])
    mats = []
    for f in range(t):
        for r in LIFT_ROTATIONS:
            ext = np.eye(4)
            ext[:3, :3] = r
            ext[:3, 3] = (1.0 * f, 0.5 * f, 0.0)   # frame 1: a dyadic sideways / upward step
            mats.append(k @ ext)
    s = len(mats)
    return dict(name=name, t=t, nv=len(LIFT_ROTATIONS), flip=flip, l2i=np.array(mats),
                scale=a['scale'], crop=a['crop'],
                meta=dict(ori_lidar2img=np.array(mats), input_shape=LIFT_IN_HW,
                          img_shape=[(60, LIFT_IMG_W, 3)] * s,
                          scale_factor=np.full(4, a['scale'], dtype=f32),
                          img_crop_offset=list(a['crop']), flip=flip))


def lift_points():
    """Voxel centres in the anchor order: z-major, then y, then x fastest."""
    xs, ys, zs = LIFT_AXES
    zz, yy, xx = np.meshgrid(zs, ys, xs, indexing='ij')
    return np.stack([xx, yy, zz], -1).reshape(-1, 3)


def lift_coords(case, p, s, prec=f32, order=0, defects=()):
    """points_cam2img, scale, crop and flip of view s: (cx, cy, depth)."""
    a, b, d = project(case['l2i'][s], p.T, prec, order)
    sc, (crx, cry) = prec(case['scale']), (prec(case['crop'][0]), prec(case['crop'][1]))
    with np.errstate(divide='ignore', invalid='ignore'):
        if 'crop_before_scale' in defects:
            cx, cy = (a / d - crx) * sc, (b / d - cry) * sc
        else:
            cx, cy = (a / d) * sc - crx, (b / d) * sc - cry
    if case['flip']:
        cx = prec(LIFT_IN_HW[1] if 'flip_about_in_w' in defects else LIFT_IMG_W) - cx
    return cx, cy, d


def lift_tap(c, size, norm, away=False):
    """nearest_index: normalise by the padded size, unnormalise with align_corners=True."""
    with np.errstate(invalid='ignore'):
        g = (c / f32(norm)) * f32(2) - f32(1)
        return round_nearest(((g + f32(1)) * f32(0.5)) * f32(size - 1), away), \
            ((g + f32(1)) * f32(0.5)) * f32(size - 1)


def lift_view(case, p, s, defects=()):
    """The kernel's per-view decisions: validity, the tap and whether it lies on the map."""
    in_h, in_w = LIFT_IN_HW
    hf, wf = LIFT_FEAT_HW
    cx, cy, d = lift_coords(case, p, s, defects=defects)
    with np.errstate(invalid='ignore'):
        x_lo = cx >= 0 if 'x_lo' in defects else cx > 0
        x_hi = cx <= in_w if 'x_hi' in defects else cx < in_w
        y_lo = cy >= 0 if 'y_lo' in defects else cy > 0
        y_hi = cy <= in_h if 'y_hi' in defects else cy < in_h
        d_ok = d >= 0 if 'depth_nonstrict' in defects else d > 0
        valid = x_lo & x_hi & y_lo & y_hi & d_ok
        away = 'round_half_away' in defects
        sx, fx = lift_tap(cx, wf, in_w, away)
        sy, fy = lift_tap(cy, hf, in_h, away)
        inside = (sx >= 0) & (sx < wf) & (sy >= 0) & (sy < hf)
    return dict(cx=cx, cy=cy, d=d, valid=valid, sx=sx, sy=sy, fx=fx, fy=fy, inside=inside)


def lift_restate(case, feats, agg, defects=()):
    """lift_voxel_kernel in numpy (fp64 sums of the exact features): [C(*T), Nx, Ny, Nz]."""
    p = lift_points()
    c = feats.shape[1]
    hf, wf = LIFT_FEAT_HW
    sums, counts = [], []
    for f in range(case['t']):
        acc = np.zeros((len(p), c))
        n = np.zeros(len(p), dtype=np.int64)
        for v in range(case['nv']):
            s = f * case['nv'] + v
            r = lift_view(case, p, s, defects)
            take = r['valid'] & r['inside']
            n += take if 'count_in_range_only' in defects else r['valid']
            idx = (np.where(take, r['sy'], 0) * wf + np.where(take, r['sx'], 0)).astype(np.int64)
            acc += np.where(take[:, None], feats[s].reshape(c, hf * wf).T[idx], 0.0)
        sums.append(acc)
        counts.append(n)
    den = (lambda n: n) if 'no_clamp' in defects else (lambda n: np.maximum(n, 1))
    with np.errstate(divide='ignore', invalid='ignore'):
        if agg == 'mean':
            out = sum(sums) / den(sum(counts))[:, None]
        else:
            out = np.concatenate([a / den(n)[:, None] for a, n in zip(sums, counts)], 1)
    nx, ny, nz = LIFT_N_VOXELS
    return out.T.reshape(-1, nz, ny, nx).transpose(0, 3, 2, 1)


def lift_feats(case, c, seed=3):
    """Multiples of 1/16 in [-8, 8): sums of up to 2 T of them are exact in fp32, and two taps
    of one map almost never hold the same channel vector."""
    rng = np.random.RandomState(seed)
    s = case['t'] * case['nv']
    hf, wf = LIFT_FEAT_HW
    return torch.from_numpy((rng.randint(-128, 128, (s, c, hf, wf)) / 16).astype(f32))


def lift_oracle(case, feats, agg):
    """oracle.multiview_lift with fp64 features and the reference's fp32 geometry."""
    pts = torch.from_numpy(lift_points())
    meta = case['meta']
    l2i = [torch.tensor(m, dtype=torch.float32) for m in case['l2i']]
    return O.multiview_lift(feats.double(), pts, LIFT_N_VOXELS, l2i, case['nv'], case['t'],
                            pts.new_tensor(meta['scale_factor'][:2]),
                            pts.new_tensor(meta['img_crop_offset']), case['flip'],
                            meta['input_shape'], meta['img_shape'], agg)


def lift_inventory(case):
    """Voxel-views at each edge kind (the other validity conditions holding), and voxels at the
    aggregation edges."""
    p = lift_points()
    in_h, in_w = LIFT_IN_HW
    inv = dict.fromkeys(('cx=0', 'cx=in_w', 'cy=0', 'cy=in_h', 'depth=0', 'behind_on_image',
                         'tie_x', 'tie_y'), 0)
    counts = []
    for f in range(case['t']):
        n = np.zeros(len(p), dtype=np.int64)
        for v in range(case['nv']):
            r = lift_view(case, p, f * case['nv'] + v)
            cx, cy, d = r['cx'], r['cy'], r['d']
            with np.errstate(invalid='ignore'):
                xin, yin = (cx > 0) & (cx < in_w), (cy > 0) & (cy < in_h)
                inv['cx=0'] += int(((cx == 0) & yin & (d > 0)).sum())
                inv['cx=in_w'] += int(((cx == in_w) & yin & (d > 0)).sum())
                inv['cy=0'] += int(((cy == 0) & xin & (d > 0)).sum())
                inv['cy=in_h'] += int(((cy == in_h) & xin & (d > 0)).sum())
                inv['depth=0'] += int((d == 0).sum())
                inv['behind_on_image'] += int(((d < 0) & xin & yin).sum())
            inv['tie_x'] += int((r['valid'] & tie_splits(r['fx'])).sum())
            inv['tie_y'] += int((r['valid'] & tie_splits(r['fy'])).sum())
            # a valid view's tap always lies on the map: c in (0, size) maps into (0, S - 1)
            assert bool(r['inside'][r['valid']].all())
            n += r['valid']
        counts.append(n)
    counts = np.stack(counts)
    inv['frame_without_view'] = int(((counts == 0) & (counts.sum(0) > 0)).any(0).sum())
    inv['unseen'] = int((counts.sum(0) == 0).sum())
    inv['flip_img_w!=in_w'] = int(case['flip'] and LIFT_IMG_W != in_w)
    return inv


LIFT_EXPECT = ('cx=0', 'cx=in_w', 'cy=0', 'cy=in_h', 'depth=0', 'behind_on_image', 'tie_x',
               'tie_y', 'unseen')
# decisions a wrong rule would change; the last two are kept apart below
LIFT_DEFECTS = ('x_lo', 'x_hi', 'y_lo', 'y_hi', 'round_half_away', 'flip_about_in_w',
                'crop_before_scale', 'no_clamp')
# Equivalent rules, shown equal on the cases rather than separated: depth 0 makes cx and cy
# infinite or NaN, which fails the image bounds, so `d > 0` and `d >= 0` decide alike; and a
# valid view's tap always lies on the map (lift_inventory asserts it), so counting a view only
# when its tap is in range changes nothing.
LIFT_EQUIVALENT = ('depth_nonstrict', 'count_in_range_only')
LIFT_GRID = [(name, t, flip) for name in LIFT_CASES for t in (1, 2) for flip in (False, True)]


def _lift_id(c):
    return f'{c[0]}-T{c[1]}' + ('-flip' if c[2] else '')


@pytest.mark.parametrize('spec', LIFT_GRID, ids=_lift_id)
def test_lift_geometry_exact(spec):
    """fp32 in two summation orders and fp64 give the same cx, cy, depth and tap coordinate at
    every voxel and view; the voxel centres are the library's own."""
    from depth_from_motion_b200.modules import aligned_voxel_centers
    for mine, lib in zip(LIFT_AXES, aligned_voxel_centers(LIFT_N_VOXELS, LIFT_RANGE)):
        assert np.array_equal(mine, lib.numpy())
    case = lift_case(*spec)
    p = lift_points()
    in_h, in_w = LIFT_IN_HW
    hf, wf = LIFT_FEAT_HW
    for s in range(len(case['l2i'])):
        res = [lift_coords(case, p, s, prec, order)
               for prec, order in ((f32, 0), (f32, 1), (np.float64, 0))]
        for k in range(3):
            assert agree(*(r[k] for r in res)), (s, k)
        with np.errstate(invalid='ignore'):
            taps = [lift_tap(r[0], wf, in_w)[1] for r in res[:2]] + \
                [(res[2][0] / in_w * 2 - 1 + 1) / 2 * (wf - 1)]
            taps_y = [lift_tap(r[1], hf, in_h)[1] for r in res[:2]] + \
                [(res[2][1] / in_h * 2 - 1 + 1) / 2 * (hf - 1)]
        assert agree(*taps) and agree(*taps_y), s


@pytest.mark.parametrize('spec', LIFT_GRID, ids=_lift_id)
def test_lift_cases_hit_the_edges(spec):
    case = lift_case(*spec)
    inv = lift_inventory(case)
    print(f'\nlift {_lift_id(spec)}: {inv}')
    for k in LIFT_EXPECT:
        assert inv[k] > 0, (k, inv)
    if case['t'] == 2:
        assert inv['frame_without_view'] > 0, inv
    if case['flip']:
        assert inv['flip_img_w!=in_w'] == 1


@pytest.mark.parametrize('spec', LIFT_GRID, ids=_lift_id)
@pytest.mark.parametrize('agg', ['mean', 'concat'])
def test_lift_restatement_equals_oracle_and_defects_separate(spec, agg):
    """The numpy restatement of the kernel equals oracle.multiview_lift (and its per-view
    point_sample masks) exactly; each planted defect changes at least one element where it
    applies."""
    case = lift_case(*spec)
    feats = lift_feats(case, 8)
    want = lift_restate(case, feats.double().numpy(), agg)
    ref = lift_oracle(case, feats, agg).numpy()
    assert np.array_equal(want, ref)
    pts = torch.from_numpy(lift_points())
    for s in range(len(case['l2i'])):
        _, valid = O.point_sample(feats[s][None].double(), pts,
                                  torch.tensor(case['l2i'][s], dtype=torch.float32),
                                  pts.new_tensor(case['meta']['scale_factor'][:2]),
                                  pts.new_tensor(case['crop']), case['flip'], LIFT_IN_HW,
                                  (60, LIFT_IMG_W), aligned=False, valid_flag=True)
        assert np.array_equal(valid.numpy(), lift_view(case, lift_points(), s)['valid'])
    rows = []
    for defect in LIFT_DEFECTS + LIFT_EQUIVALENT:
        if defect == 'flip_about_in_w' and not case['flip']:
            continue
        if defect == 'crop_before_scale' and case['scale'] == 1:
            continue
        got = lift_restate(case, feats.double().numpy(), agg, (defect,))
        changed = int((~((got == ref) | (np.isnan(got) & np.isnan(ref)))).any(0).sum())
        rows.append((defect, changed))
    print(f'\nlift {_lift_id(spec)} {agg}: defect -> voxels changed {rows}')
    for defect, changed in rows:
        assert (changed == 0) == (defect in LIFT_EQUIVALENT), (defect, changed)


def run_lift(spec, agg, c, monkeypatch):
    from depth_from_motion_b200 import capi, modules
    case = lift_case(*spec)
    feats = lift_feats(case, c)
    ref = lift_oracle(case, feats, agg).float()
    args = (case['meta'], LIFT_N_VOXELS, LIFT_RANGE, case['nv'], case['t'], agg)
    dev = feats.cuda()
    L = capi.lib()
    got = {}
    for cl in (False, True):
        # separate allocations: the pointer-table entry
        views = [dev[s].clone() for s in range(dev.shape[0])]
        got['views' + ('_cl' if cl else '')] = modules.multiview_lift(views, *args,
                                                                      channels_last=cl)
        # the same call routed to the contiguous entry (table[0] is the start of `dev`)
        name = 'dfm_multiview_lift_views' + ('_cl' if cl else '')
        with monkeypatch.context() as mp:
            mp.setattr(L, name, lambda desc, table, *rest, fn=getattr(L, name.replace(
                '_views', '')): fn(desc, ctypes.c_void_p(table[0]), *rest))
            got['contiguous' + ('_cl' if cl else '')] = modules.multiview_lift(
                dev, *args, channels_last=cl)
    capi.sync_check()
    bad = {k: int((v.cpu() != ref).any(0).sum()) for k, v in got.items()}
    print(f'\nlift {_lift_id(spec)} {agg} C={c}: edges {lift_inventory(case)}, '
          f'mismatching voxels {bad}')
    for k, v in got.items():
        assert v.shape == ref.shape and torch.equal(v.cpu(), ref), (k, bad[k])
    assert float(ref.abs().sum()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize('spec', LIFT_GRID, ids=_lift_id)
@pytest.mark.parametrize('agg', ['mean', 'concat'])
def test_lift_bit_exact(spec, agg, monkeypatch):
    """Every lift entry (NCDHW and channels-last, pointer table and contiguous) equals the fp64
    oracle rounded to fp32, at every voxel."""
    run_lift(spec, agg, 64, monkeypatch)


@pytest.mark.gpu
def test_lift_bit_exact_128_channels(monkeypatch):
    """C = 128, the most the warp-per-voxel kernel's four per-lane accumulators hold."""
    run_lift(('aug', 2, True), 'concat', 128, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize('channels_last', [False, True])
def test_lift_refuses_160_channels_before_launch(channels_last):
    from depth_from_motion_b200 import capi, modules
    case = lift_case('plain', 1, False)
    feats = lift_feats(case, 160).cuda()
    nx, ny, nz = LIFT_N_VOXELS
    out = torch.full((nx, ny, nz, 160), 7.0, device='cuda')
    with pytest.raises(RuntimeError, match='at most 128 channels'):
        modules.multiview_lift(feats, case['meta'], LIFT_N_VOXELS, LIFT_RANGE, case['nv'],
                               case['t'], 'mean', out=out if channels_last else None,
                               channels_last=channels_last)
    capi.sync_check()
    assert bool((out == 7.0).all())   # nothing was written


# ---------------------------------------------------------------------------------------------
# FrustumToVoxel gather (frustum_gather_kernel, csrc/frustum_kernels.cuh)
# ---------------------------------------------------------------------------------------------
# pad_w - 1 and pad_h - 1 are powers of two, so u / (pad_w - 1) is exact; Wo - 1 = 32 and
# Ho - 1 = 16 make the stereo and semantic taps exact too
FR_PAD = (65, 129)
FR_VOL = (8, 17, 33)     # D, Ho, Wo of the stereo volume; the semantic map is Ho x Wo
FR_P = [[2., 0, 64, 0], [0, 2., 32, 0], [0, 0, 1, 0], [0, 0, 0, 1]]
# pseudo-lidar x is the rect depth: -2 .. 2; u = 64 - 2 y / x spans 0 .. 129 at x = 1
FR_AXES = (axis(-2, 1, 5), axis(-34, .5, 137), axis(-17, .5, 68))
FR_DEPTH = dict(mode='UD', num_bins=4 * FR_VOL[0], depth_min=1.0, depth_max=2.0,
                downsample_factor=4)
FR_VARIANTS = dict(default={}, stereo_atten=dict(stereo_atten_feat=True, sem_atten_feat=False),
                   no_img=dict(cat_img_feature=False, stereo_atten_feat=True))


def fr_coordinates():
    xs, ys, zs = (torch.from_numpy(a) for a in FR_AXES)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    return torch.stack([xx, yy, zz], -1)


def fr_restate(prec=f32, order=0, defects=()):
    """frustum_gather_kernel's phase A: (u, v, normalised x / y / depth, valid2d, valid),
    each [nz, ny, nx]."""
    c3d = fr_coordinates().numpy()
    x, y, z = c3d[..., 0], c3d[..., 1], c3d[..., 2]
    pu, pv, pw = project(np.array(FR_P), (-y, -z, x), prec, order)
    ph, pwid = prec(FR_PAD[0]), prec(FR_PAD[1])
    dmin, dspan = prec(FR_DEPTH['depth_min']), prec(FR_DEPTH['depth_max'] - FR_DEPTH['depth_min'])
    one, two = prec(1), prec(2)
    with np.errstate(divide='ignore', invalid='ignore'):
        u, v = pu / pw, pv / pw
        nxn = u / (pwid - one) * two - one
        nyn = v / (ph - one) * two - one
        nzn = (x.astype(prec) - dmin) / dspan * two - one
        u_lo = u > 0 if 'u_lo' in defects else u >= 0
        u_hi = u < pwid if 'u_hi' in defects else u <= pwid
        v_lo = v > 0 if 'v_lo' in defects else v >= 0
        v_hi = v < ph if 'v_hi' in defects else v <= ph
        d_lo = nzn > -1 if 'depth_lo' in defects else nzn >= -1
        d_hi = nzn < 1 if 'depth_hi' in defects else nzn <= 1
    valid2d = u_lo & u_hi & v_lo & v_hi
    return dict(u=u, v=v, pw=pw, nxn=nxn, nyn=nyn, nzn=nzn, valid2d=valid2d,
                valid=valid2d & d_lo & d_hi)


FR_DEFECTS = ('u_lo', 'u_hi', 'v_lo', 'v_hi', 'depth_lo', 'depth_hi')


def fr_inventory():
    r = fr_restate()
    u, v, nzn, v2 = r['u'], r['v'], r['nzn'], r['valid2d']
    with np.errstate(invalid='ignore'):
        uin, vin = (u > 0) & (u < FR_PAD[1]), (v > 0) & (v < FR_PAD[0])
        return {'u=0': int(((u == 0) & vin).sum()), 'u=pad_w': int(((u == FR_PAD[1]) & vin).sum()),
                'v=0': int(((v == 0) & uin).sum()), 'v=pad_h': int(((v == FR_PAD[0]) & uin).sum()),
                'depth=-1': int((v2 & (nzn == -1)).sum()), 'depth=+1': int((v2 & (nzn == 1)).sum()),
                'depth=0': int((r['pw'] == 0).sum()),
                'behind_on_image': int((v2 & (r['pw'] < 0)).sum()),
                'valid': int(r['valid'].sum())}


def test_frustum_geometry_exact():
    """The projection, the pixel and the normalised coordinates agree bit for bit in fp32
    (two summation orders) and fp64; the voxel axes are separable as the module requires."""
    res = [fr_restate(prec, order) for prec, order in ((f32, 0), (f32, 1), (np.float64, 0))]
    for k in ('u', 'v', 'pw', 'nxn', 'nyn', 'nzn', 'valid2d', 'valid'):
        assert agree(*(r[k] for r in res)), k
    from depth_from_motion_b200.modules import FrustumToVoxel
    got = FrustumToVoxel._separable_centres(fr_coordinates())
    assert all(np.array_equal(a, b.numpy()) for a, b in zip(FR_AXES, got))


def test_frustum_case_hits_the_edges():
    inv = fr_inventory()
    print(f'\nfrustum: {inv}')
    assert all(n > 0 for n in inv.values()), inv


def test_frustum_restatement_equals_oracle_and_defects_separate():
    norm, valid2d, valid = O.frustum_grid(fr_coordinates(), FR_P, FR_PAD, FR_DEPTH)
    r = fr_restate()
    for k, i in (('nxn', 0), ('nyn', 1), ('nzn', 2)):
        assert agree(norm[..., i].numpy(), r[k]), k
    assert np.array_equal(valid2d.numpy(), r['valid2d'])
    assert np.array_equal(valid.numpy().astype(bool), r['valid'])
    rows = []
    for defect in FR_DEFECTS:
        d = fr_restate(defects=(defect,))
        rows.append((defect, int((d['valid2d'] != r['valid2d']).sum() +
                                 (d['valid'] != r['valid']).sum())))
    print(f'\nfrustum: defect -> mask decisions changed {rows}')
    assert all(n > 0 for _, n in rows), rows


def fr_inputs(seed=61):
    rng = np.random.RandomState(seed)
    d, ho, wo = FR_VOL
    t = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(f32))  # noqa: E731
    return dict(stereo=t(1, 32, d, ho, wo), cost=t(1, 1, d, ho, wo) * 2, sem=t(1, 32, ho, wo),
                weight=t(32, 64, 3, 3, 3) * 0.05)


def fr_reference(inp, sm, stereo_atten_feat=False, sem_atten_feat=True, cat_img_feature=True):
    """feature_transformation.py:84-160 in fp64 on the oracle's grid (oracle.frustum_grid).
    Depth-0 voxels have a non-finite sample point and both masks 0; the point is moved off
    the volume so that the masked sample is 0, not NaN * 0."""
    norm, valid2d, valid = O.frustum_grid(fr_coordinates(), FR_P, FR_PAD, FR_DEPTH)
    g = norm.double()
    g[~torch.isfinite(g).all(-1)] = 2.0
    g = g[None]
    valid, valid2d = valid.double()[None, None], valid2d.double()[None, None]
    vox = F.grid_sample(inp['stereo'].double(), g, align_corners=True) * valid
    disp = None
    if stereo_atten_feat or (sem_atten_feat and cat_img_feature):
        disp = F.grid_sample(sm, g, align_corners=True) * valid
        if stereo_atten_feat:
            vox = vox * disp
    if cat_img_feature:
        g2 = g.clone()
        g2[..., 2] = 0
        v2 = F.grid_sample(inp['sem'].double().unsqueeze(2), g2, align_corners=True) * valid2d
        if sem_atten_feat:
            v2 = v2 * disp
        vox = torch.cat([vox, v2], 1)
    return vox[0]


@pytest.mark.gpu
@pytest.mark.parametrize('fused', [True, False], ids=['fused_softmax', 'materialised_softmax'])
@pytest.mark.parametrize('variant', list(FR_VARIANTS))
def test_frustum_gather_exact_masks(variant, fused):
    """debug_tensor('vox') against the fp64 reference at every voxel, edges included: the
    zero / non-zero decision of each half is identical and the values are within GATHER_TOL.
    The stereo and semantic tap coordinates are exact here, but those of the x4 depth
    distribution cannot be: its 4 Ho - 1 rows are odd in number, so v / 64 * 67 rounds in fp32
    and moves the attention's weights by up to an ulp of the coordinate (about 4e-6).  That,
    the fp32 blends and the fused path's fast exponential are what GATHER_TOL bounds (worst
    measured on an H100: 1.3e-6)."""
    from depth_from_motion_b200 import capi, modules
    from tests.test_stage_layers import GATHER_TOL
    kw = FR_VARIANTS[variant]
    inp = fr_inputs()
    cat = kw.get('cat_img_feature', True)
    cin = 64 if cat else 32
    m = modules.FrustumToVoxel(**kw)
    m.load_state_dict({'voxel_convs.0.0.conv.weight': inp['weight'][:, :cin],
                       'voxel_convs.0.0.gn.weight': torch.ones(32),
                       'voxel_convs.0.0.gn.bias': torch.zeros(32)}, strict=True)
    m = m.cuda().eval()
    m.coordinates_3d = fr_coordinates()
    m.depth_cfg = FR_DEPTH
    _, sm, _ = O.depth_head_forward(inp['cost'], O.depth_samples(FR_DEPTH), 4)
    _, sm64, _ = O.depth_head_forward(inp['cost'].double(), O.depth_samples(FR_DEPTH).double(), 4)
    dist = modules.CostLogits(inp['cost'].cuda()) if fused else sm.cuda()
    metas = [dict(cam2img=FR_P, pad_shape=FR_PAD + (3,))]
    with torch.no_grad():
        m(inp['stereo'].cuda(), dist, metas, inp['sem'].cuda() if cat else None)
    nz, ny, nx = (len(a) for a in FR_AXES[::-1])
    got = m.debug_tensor('vox', (nz, ny, nx, cin)).movedim(-1, 0).double().cpu()
    capi.sync_check()
    ref = fr_reference(inp, sm64, **kw)
    assert got.shape == ref.shape
    r = fr_restate()
    rows = {}
    for half, mask in (('stereo', r['valid']),
                       ('sem', r['valid'] if kw.get('sem_atten_feat', True) else r['valid2d'])):
        if half == 'sem' and not cat:
            continue
        sl = slice(0, 32) if half == 'stereo' else slice(32, 64)
        gz, rz = (got[sl] == 0).all(0).numpy(), (ref[sl] == 0).all(0).numpy()
        # masked voxels are zero; so are the few whose depth-distribution taps all fall off the
        # x4 softmax volume (v = pad_h: (65 / 64) * 67 > 67) where the attention multiplies
        assert rz[~mask].all() and not rz[mask].all(), half
        err = float((got[sl] - ref[sl]).abs().max() / ref[sl].abs().max())
        rows[half] = dict(mask_mismatches=int((gz != rz).sum()), err=err)
    print(f'\nfrustum {variant} {"fused" if fused else "materialised"}: edges {fr_inventory()}, '
          f'{rows} (value bound {GATHER_TOL:.0e})')
    for half, row in rows.items():
        assert row['mask_mismatches'] == 0, (half, row)
        assert row['err'] <= GATHER_TOL, (half, row)
    m.release()


# ---------------------------------------------------------------------------------------------
# voxel_sample (voxel_sample_kernel, csrc/voxel_sample_api.inc)
# ---------------------------------------------------------------------------------------------
# 16 x 16 x 2 unit voxels: idx / n is exact for power-of-two n; with n = 2 the unnormalised z
# index is idx / 2, so the centres at z = 0.5 and z = -1.5 land on 0.5 and -0.5, where half-even
# and half-away rounding pick different taps (for n = 2^k > 2 the only tie, 2^(k-1) - 0.5,
# rounds to the same even tap under both rules)
VS_RANGE, VS_SIZE, VS_N = [0., -8., -1., 16., 8., 1.], [1., 1., 1.], (16, 16, 2)
VS_PAD, VS_IMG, VS_DF = (32, 64), (30, 60), 4
VS_DEPTHS = torch.tensor([1., 2., 4., 8.]).repeat_interleave(VS_DF)   # [::4] = 1, 2, 4, 8
VS_CASES = {
    'plain': dict(f=8., c=(32., 16.), t=(0., 0., 0.), scale=1., crop=(0., 0.), flip=False),
    'aug': dict(f=16., c=(64., 32.), t=(0.5, 0., 0.), scale=.5, crop=(4., 2.), flip=True),
}


def vs_args(name):
    a = VS_CASES[name]
    k = np.array([[a['f'], 0, a['c'][0], 0], [0, a['f'], a['c'][1], 0], [0, 0, 1, 0],
                  [0, 0, 0, 1]])
    ext = np.eye(4)
    ext[:3, :3] = LIFT_ROTATIONS[0]
    ext[:3, 3] = a['t']
    proj = torch.tensor(k @ ext, dtype=torch.float32)
    return (VS_RANGE, VS_SIZE, VS_DEPTHS, proj, VS_DF, torch.tensor([a['scale']] * 2),
            torch.tensor(a['crop']), a['flip'], VS_PAD, VS_IMG)


def vs_restate(name, prec=f32, order=0, defects=()):
    """voxel_sample_kernel's coordinate chain: the unnormalised (x, y, z) index, [3, D, H, W]."""
    a = VS_CASES[name]
    _, _, depths, proj, df, _, _, flip, (h, w), img = vs_args(name)
    ho, wo = round(h / df), round(w / df)
    dep, v, u = np.meshgrid(depths[::df].numpy(), np.arange(ho) * df, np.arange(wo) * df,
                            indexing='ij')
    u, v, dep = u.astype(prec), v.astype(prec), dep.astype(prec)
    if flip:
        u = prec(w if 'flip_about_pad_w' in defects else img[1]) - u
    sc, crx, cry = prec(a['scale']), prec(a['crop'][0]), prec(a['crop'][1])
    if 'crop_after_scale' in defects:
        u, v = u / sc + crx, v / sc + cry
    else:
        u, v = (u + crx) / sc, (v + cry) / sc
    pinv = np.linalg.inv(proj.double().numpy()).astype(f32)
    cam = project(pinv, (u * dep, v * dep, dep), prec, order)
    out = []
    for r in range(3):
        lo, vs, n = prec(VS_RANGE[r]), prec(VS_SIZE[r]), VS_N[r]
        inv_vs = prec(1) / vs
        inv_ext = prec(1) / ((prec(VS_RANGE[3 + r]) - lo) / vs)
        idx = (cam[r] - lo) * inv_vs - prec(0.5)
        g = idx * inv_ext * prec(2) - prec(1)
        out.append((g + prec(1)) * prec(0.5) * prec(n - 1))
    return np.stack(out)


VS_DEFECTS = ('index_lo', 'index_hi', 'round_half_away', 'flip_about_pad_w', 'crop_after_scale')


def vs_nearest(name, vox, defects=()):
    """voxel_sample(aligned=False) in numpy: [C, D, H, W]; a read past the array (only a
    planted bound can make one) gives NaN."""
    f = vs_restate(name, defects=defects)
    i = round_nearest(f, 'round_half_away' in defects)
    n = np.array(VS_N)[:, None, None, None]
    lo = i > 0 if 'index_lo' in defects else i >= 0
    hi = i <= n if 'index_hi' in defects else i < n
    ok = (lo & hi).all(0)
    pad = np.pad(vox, ((0, 0), (0, 1), (0, 1), (0, 1)), constant_values=np.nan)
    ii = np.where(ok, i, 0).astype(np.int64)
    return np.where(ok, pad[:, ii[0], ii[1], ii[2]], 0.0)


def vs_features(seed=17, c=4):
    rng = np.random.RandomState(seed)
    return torch.from_numpy((rng.randint(1, 256, (1, c) + VS_N) / 16).astype(f32))


def vs_inventory(name):
    f = vs_restate(name)
    i = round_nearest(f)
    n = np.array(VS_N)[:, None, None, None]
    ok = ((i >= 0) & (i < n)).all(0)
    return {'tie_splits': int((tie_splits(f) & ok).sum()),
            'index_0': int((ok & (i == 0).any(0)).sum()),
            'index_n-1': int((ok & (i == n - 1).any(0)).sum()),
            'off_grid': int((~ok).sum()), 'on_grid': int(ok.sum())}


@pytest.mark.parametrize('name', list(VS_CASES))
def test_voxel_sample_geometry_exact(name):
    """The inverse projection is exact in fp32 (torch.inverse, which the oracle uses, equals
    the fp64 inverse), and the unnormalised index agrees in fp32 (two orders) and fp64."""
    proj = vs_args(name)[3]
    assert np.array_equal(torch.inverse(proj).numpy(), np.linalg.inv(proj.double().numpy()))
    assert agree(vs_restate(name, f32, 0), vs_restate(name, f32, 1),
                 vs_restate(name, np.float64, 0))
    inv = vs_inventory(name)
    print(f'\nvoxel_sample {name}: {inv}')
    assert all(v > 0 for v in inv.values()), inv


@pytest.mark.parametrize('name', list(VS_CASES))
def test_voxel_sample_restatement_equals_oracle_and_defects_separate(name):
    vox = vs_features()
    ref = O.voxel_sample(vox, *vs_args(name), aligned=False)[0].numpy()
    assert np.array_equal(vs_nearest(name, vox[0].numpy()), ref)
    rows = []
    for defect in VS_DEFECTS:
        if defect in ('flip_about_pad_w', 'crop_after_scale') and not VS_CASES[name]['flip']:
            continue
        got = vs_nearest(name, vox[0].numpy(), (defect,))
        rows.append((defect, int((got != ref).any(0).sum())))
    print(f'\nvoxel_sample {name}: defect -> samples changed {rows}')
    assert all(n > 0 for _, n in rows), rows


@pytest.mark.gpu
@pytest.mark.parametrize('aligned', [False, True], ids=['nearest', 'trilinear'])
@pytest.mark.parametrize('name', list(VS_CASES))
def test_voxel_sample_exact_geometry(name, aligned):
    """Nearest: equal to the oracle at every sample.  Trilinear: the existing 1e-4 bound."""
    from depth_from_motion_b200 import capi, modules
    vox = vs_features()
    args = vs_args(name)
    ref = O.voxel_sample(vox, *args, aligned=aligned)
    got = modules.voxel_sample(vox.cuda(), *args, aligned=aligned).cpu()
    capi.sync_check()
    assert got.shape == ref.shape
    bad = int((got != ref).any(1).sum())
    err = float((got - ref).abs().max() / ref.abs().max())
    print(f'\nvoxel_sample {name} {"trilinear" if aligned else "nearest"}: '
          f'edges {vs_inventory(name)}, mismatching samples {bad}, err {err:.2e}')
    if aligned:
        assert err < 1e-4
    else:
        assert bad == 0
