"""Layer-by-layer parity of the stages after the backbone against an fp64 reference: the Waymo
necks (DfMNeck, OutdoorImVoxelNeck), FrustumToVoxel, BEVHourglass and LIGAAnchor3DHead.

The end-to-end tests hold these stages to the 1e-3 bar, about what one lost bf16 product term,
a wrong normalisation of one channel block or a stale tile costs the final map.  Here every
conv is judged on its own, as test_backbone_layers.py does for the backbone:

* one forward; every raw conv output is read back through the module's ``debug_tensor``;
* each layer's input is rebuilt in float64 from the GPU's OWN upstream raw outputs: BatchNorm
  is static, GroupNorm statistics are recomputed in float64 from the whole GPU tensor, and ReLU
  and residuals are applied as ``oracle.dfm_oracle`` does (``_res_module`` / ``_neck_tower``,
  ``frustum_to_voxel_forward``, ``bev_hourglass_forward``, ``liga_anchor3d_head_forward``);
* the conv runs in float64 and is compared with the GPU's raw output of that layer.

Tensor-core layers are held to ``max(K_E3 e3, floor)`` with the bound at least SEPARATION times
below ``e2`` (tests/layer_check.py), in the normalised max-norm and element-wise on the shell:
first and last index of every axis, the ragged last tile, both sides of every tile seam of the
K-outer kernel (16 x 8 voxels) and of every window seam along its marched axis.  The fp32
CUDA-core layers (the BEV stride-2 and transposed convs, everything under ``conv_impl='simt'``)
have no split and are held to the accumulation floor alone, which must also stay SEPARATION
times below the e2 the layer would have on the tensor-core path.  Element-wise fp32 stages (the
neck gate, GroupNorm + ReLU + AvgPool of FrustumToVoxel, the BEV emits) are compared with their
fp64 restatement on the GPU's own inputs.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O
from tests import layer_check as LC
from tests.layer_check import SEPARATION, elementwise_errors, layer_bound

# fp32 accumulation floor of these stages: the necks' K-outer kernel keeps its accumulators in
# registers across up to 8 channel groups (K = 27 * 256 = 6912); on an H100 the 256-channel
# layers reach 1.54x the backbone's 4 sqrt(K) u and 6.7x e3, so the floor is 8 sqrt(K) u here
FLOOR_C = 8.0
EW_TOL = 1e-5           # element-wise fp32 stages, relative to the max of the reference
# the frustum gather samples with fp32 coordinates on both sides, computed in a different
# order; 3x the worst error measured on an H100 (8.4e-6 at the KITTI grid)
GATHER_TOL = 3e-5
TC_KINDS = ('conv_tc_neck', 'conv2d_tc', 'conv_tck', 'conv_tc', 'conv_tc_ks')

# ---------------------------------------------------------------------------------------------
# BEV necks (csrc/neck_api.inc): 9 convs per tower
# ---------------------------------------------------------------------------------------------
NECK_KEYS = ('0.conv0', '0.conv1', '1', '2.conv0', '2.conv1', '3', '4.conv0', '4.conv1', '5')
NECK_ZMODE = ('s1', 's1', 'z2', 's1', 's1', 'z2', 's1', 's1', 'p0')
NECK_TILE = (16, 8)      # conv_tc_neck.cuh NK_BY (along Nx) x NK_BX (along Ny)
# the benchmarked Waymo grid: x / y crops cover the first and ragged last tile and interior
# seams on both axes (16 | 8-aligned boundaries at 112 / 128 and 144 / 152 / 160)
WAYMO_CROPS_X = ((0, 20), (104, 136), (200, 220))
WAYMO_CROPS_Y = ((0, 12), (144, 164), (288, 300))


def neck_geom(i, region=None):
    """Geometry of neck layer i: stride (1,1,2) on down1 / down3, pad (1,1,0) on out5."""
    return dict(stride=(1, 1, 2) if NECK_ZMODE[i] == 'z2' else 1,
                pad=(1, 1, 0) if NECK_ZMODE[i] == 'p0' else 1, region=region)


def neck_layers(x, p, tower, fetch):
    """(layer, input) of the nine convs of one tower in forward order (neck_tower_forward =
    oracle._neck_tower / _res_module), inputs rebuilt in fp64 from fetch(i), the raw output of
    layer i."""
    def bn(i):
        return folded_bn(fetch(i), p, f'{tower}.{NECK_KEYS[i]}.bn')
    yield 0, x
    yield 1, F.relu(bn(0))
    yield 2, F.relu(x + bn(1))
    a3 = F.relu(bn(2))
    yield 3, a3
    yield 4, F.relu(bn(3))
    yield 5, F.relu(a3 + bn(4))
    a6 = F.relu(bn(5))
    yield 6, a6
    yield 7, F.relu(bn(6))
    yield 8, F.relu(a6 + bn(7))


def folded_bn(x, p, prefix):
    """Eval-mode BatchNorm3d as the library applies it: folded once into a per-channel fp32
    scale and shift (neck_layer_try_fold), then x * scale + shift.  The fp32 rounding of the
    folded parameters is part of the model the kernels run, not an error of the conv that
    consumes them, so the reference input carries it too."""
    s = p[prefix + '.weight'] / torch.sqrt(p[prefix + '.running_var'] + 1e-5)
    sh = (p[prefix + '.bias'] - p[prefix + '.running_mean'] * s).float().double()
    s = s.float().double()
    return x * s[:, None, None, None] + sh[:, None, None, None]


def neck_zwindow(zo, cg):
    """Output planes per window of conv_tc_neck (neck_tc_conv): NK_ACC_COLS / NCTA planes fit."""
    zmax = 128 // (1024 // cg)
    if zo <= zmax:
        return zo
    n = -(-zo // zmax)
    return -(-zo // n)


# ---------------------------------------------------------------------------------------------
# comparison core
# ---------------------------------------------------------------------------------------------
def crop(t, region):
    """t [1, C, *S] restricted to region (per spatial axis (lo, hi) or None)."""
    return t[(slice(None), slice(None)) + tuple(slice(None) if r is None else slice(*r)
                                                for r in region)]


def axis_shell(n, tile):
    """First / last index, both sides of every tile (or window) seam and the ragged last tile."""
    i = torch.arange(n)
    sel = (i == 0) | (i == n - 1)
    if tile and tile < n:
        sel |= (i % tile == 0) | (i % tile == tile - 1)
        if n % tile:
            sel |= i >= n // tile * tile
    return sel


def shell_mask(shape, tiles, region):
    """Shell of a tensor of spatial `shape` (tile / window length per axis), on `region`."""
    sels = []
    for a, (n, t) in enumerate(zip(shape, tiles)):
        sel = axis_shell(n, t)
        sels.append(sel if region[a] is None else sel[region[a][0]:region[a][1]])
    m = torch.zeros([len(v) for v in sels], dtype=torch.bool)
    for a, sel in enumerate(sels):
        view = [1] * len(sels)
        view[a] = -1
        m = m | sel.view(view)
    return m


class Checker:
    """Collects one row per compared layer and every bound that failed."""

    def __init__(self, case):
        self.case, self.rows, self.failures, self.checked = case, [], [], set()

    def conv(self, label, got, x, w, classes, k, regions=None, tiles=None, simt=False, **g):
        """got: the GPU's raw output [1, C, *S]; x, w: the fp64 input and weight; g: geometry.
        tiles: per output axis the tile / window length of the shell check (None: no shell)."""
        regions = regions or [(None,) * (got.dim() - 2)]
        cols = {n: [] for n in ('got', 'ref', 'y3', 'y2x', 'y2w', 'sc', 'm')}
        for r in regions:
            ref = LC.conv_planes(x, w, region=r, **g)
            ys = LC.emulated_outputs(x, w, region=r, **g)
            part = dict(got=crop(got, r), ref=ref, y3=ys[0], y2x=ys[1], y2w=ys[2],
                        sc=LC.product_scale(x, w, region=r, **g))
            assert part['got'].shape == ref.shape, (label, part['got'].shape, ref.shape)
            for n, t in part.items():
                cols[n].append(t.flatten(2)[0])
            if tiles is not None:
                cols['m'].append(shell_mask(tuple(got.shape[2:]), tiles, r).flatten())
        c = {n: torch.cat(v, 1) if n != 'm' else (torch.cat(v) if v else None)
             for n, v in cols.items()}
        s = float(c['ref'].abs().max())
        e = float((c['got'] - c['ref']).abs().max()) / s
        e3, e2 = LC.norm_errors((c['y3'], c['y2x'], c['y2w']), c['ref'])
        # the fp32 CUDA-core kernels have no split: the accumulation floor alone
        bound = LC.acc_floor(k, FLOOR_C) if simt else layer_bound(e3, k, FLOOR_C)
        line = dict(layer=label, cls=' | '.join(classes), err=e, e3=e3, e2=e2, bound=bound)
        if c['m'] is not None and bool(c['m'].any()):
            m = c['m'].to(c['ref'].device)
            eg, el3, el2, elb = elementwise_errors(*(c[n][:, m] for n in
                                                     ('got', 'ref', 'y3', 'y2x', 'y2w', 'sc')), k,
                                                   FLOOR_C)
            if simt:
                elb = LC.acc_floor(k, FLOOR_C)
            line.update(shell=eg, shell_bound=elb, shell_e2=el2)
            if eg > elb:
                self.failures.append((label, 'shell element', eg, elb))
            if SEPARATION * elb > el2:
                self.failures.append((label, 'shell separation', elb, el2))
        if e > bound:
            self.failures.append((label, e, bound))
        if SEPARATION * bound > e2:
            self.failures.append((label, 'separation', bound, e2))
        self.rows.append(line)
        self.checked.update(classes)

    def elementwise(self, label, got, ref, tol=EW_TOL, cls='', excluded=None):
        e = float((got.double() - ref).abs().max()) / float(ref.abs().max())
        self.rows.append(dict(layer=label, cls=cls, err=e, bound=tol, excluded=excluded))
        if e > tol:
            self.failures.append((label, e, tol))

    def report(self, report):
        nan = float('nan')
        print(f'\n{self.case}: kernel classes launched: {sorted(report)}')
        print('case | layer | kernel | GPU err | bound | e3 | e2 | err/e3 || shell element-wise: '
              'GPU | bound | e2')
        for r in self.rows:
            extra = f" (excluded {r['excluded']})" if r.get('excluded') is not None else ''
            print(f"{self.case} | {r['layer']} | {r['cls']} | {r['err']:.2e} | {r['bound']:.2e} | "
                  f"{r.get('e3', nan):.2e} | {r.get('e2', nan):.2e} | "
                  f"{r['err'] / r.get('e3', nan):.2f} || {r.get('shell', nan):.2e} | "
                  f"{r.get('shell_bound', nan):.2e} | {r.get('shell_e2', nan):.2e}{extra}")
        print('CLASSES', ' '.join(sorted(report)))
        launched = {k.split('@')[0] for k in report if k.split('<')[0] in TC_KINDS}
        if launched - self.checked:
            self.failures.append(('kernel classes launched but not compared',
                                  sorted(launched - self.checked)))


def classes_of(report, kinds, cin, cout, modes, dims):
    """Kernel classes (names without the shape) of the profile report that computed a layer."""
    suffix = '@' + 'x'.join(str(v) for v in dims)
    out = set()
    for k in report:
        kind, _, rest = k.partition('<')
        if kind in kinds and k.endswith(suffix) and rest.split(',')[0] == f'{cin}->{cout}' \
                and rest.split(',')[1] in modes:
            out.add(k.split('@')[0])
    return sorted(out)


def profiled(fn):
    """Runs fn twice (the first call builds handles and weight images); returns the second
    call's result and its profile report."""
    from depth_from_motion_b200 import capi
    with torch.no_grad():
        fn()
        capi.sync_check()
        capi.profile_report()
        capi.profile_enable(True)
        try:
            out = fn()
            capi.sync_check()
            report = capi.profile_report()
        finally:
            capi.profile_enable(False)
    return out, report


def fp64(params, dev):
    return {k: torch.as_tensor(v).to(dev, torch.float64) for k, v in params.items()}


def _cl(t):
    """channels-last [*S, C] -> [1, C, *S] fp64"""
    return t.movedim(-1, 0)[None].double()


# ---------------------------------------------------------------------------------------------
# neck cases
# ---------------------------------------------------------------------------------------------
NECK_CASES = ('neck_dfm', 'neck_imvoxel', 'neck_dfm_mt', 'neck_imvoxel_mt',
              'waymo_dfm', 'waymo_imvoxel')


def make_neck_case(name, impl='auto'):
    """(module, input x [1, C, Nx, Ny, Nz] on the GPU, state dict)."""
    from depth_from_motion_b200 import modules
    from depth_from_motion_b200 import synthetic as syn
    from tests.util import GOLDEN, make_neck_mt_case
    dual = 'dfm' in name
    mod = (modules.DfMNeck(64, 256, num_frames=2, conv_impl=impl) if dual
           else modules.OutdoorImVoxelNeck(64, 256, conv_impl=impl))
    if name in ('neck_dfm', 'neck_imvoxel'):
        rng = np.random.RandomState(21)
        x = torch.from_numpy(np.load(os.path.join(GOLDEN, name + '.npz'))['x'])
    elif name.endswith('_mt'):
        rng, x = make_neck_mt_case(name)
    else:
        # the benchmark's input path: synthetic sample -> dfm_multiview_lift_cl, T=2 concat for
        # DfMNeck, T=1 mean for OutdoorImVoxelNeck
        t = 2 if dual else 1
        feats, meta = syn.make_waymo_sample(200, t, 5)

        class Host(modules.MultiViewDfMFeatureTransformation):
            n_voxels, voxel_range = syn.WAYMO_N_VOXELS, syn.WAYMO_RANGE
            temporal_aggregate = 'concat' if dual else 'mean'
            valid_sample, neck_3d = True, None
        with torch.no_grad():
            x = Host().feature_transformation(feats.cuda()[None], [meta], 5, t)[0]
        rng = np.random.RandomState(5)
    sd = syn.make_neck_params(rng, mod.state_dict())
    mod.load_state_dict(sd, strict=True)
    return mod.cuda().eval(), x.cuda(), sd


def run_neck_case(name, impl='auto'):
    mod, x, sd = make_neck_case(name, impl)
    _, nx, ny, nz = x.shape[1:]
    bev, report = profiled(lambda: mod(x)[0])
    p = fp64(sd, 'cuda')
    simt = impl == 'simt'
    regions = None
    if name.startswith('waymo'):
        regions = [(rx, ry, None) for rx in WAYMO_CROPS_X for ry in WAYMO_CROPS_Y]
    ck = Checker(name + ('' if impl == 'auto' else f' [{impl}]'))
    dual = 'dfm' in name
    x64 = x.double()
    raws = {}
    for tower, key in (('mono', 'mono_layers' if dual else 'model'), ('stereo', 'stereo_layers')):
        if tower == 'stereo' and not dual:
            continue
        xin = x64[:, :64] if (dual and tower == 'mono') else x64
        zs = [nz, nz]
        zs += [(nz - 1) // 2 + 1] * 3
        zs += [(zs[-1] - 1) // 2 + 1] * 3 + [1]
        c0 = xin.shape[1]    # 64, or 128 for DfMNeck's stereo tower (T = 2 concat)
        cin = [c0, c0, c0, 128, 128, 128, 256, 256, 256]
        cout = [c0, c0, 128, 128, 128, 256, 256, 256, 256]

        def fetch(i, tower=tower):
            if (tower, i) not in raws:
                raws[tower, i] = _cl(mod.debug_tensor(f'{tower}.{i}', (nx, ny, zs[i], cout[i])))
            return raws[tower, i]
        for i, xi in neck_layers(xin, p, key, fetch):
            w = p[f'{key}.{NECK_KEYS[i]}.conv.weight']
            dims = (nx, ny, zs[i])
            cls = classes_of(report, ('conv_tc_neck',), cin[i], cout[i], (NECK_ZMODE[i],), dims)
            cls += classes_of(report, ('conv_simt',), cin[i], cout[i], ('s1', 's2'), dims)
            cg = 16 if any(',g16,' in c for c in cls) else 32
            tiles = NECK_TILE + (neck_zwindow(zs[i], cg),)
            ck.conv(f'{tower}.{i}', fetch(i), xi, w, cls, LC.k_of(cin[i]), regions=regions,
                    tiles=tiles, simt=simt, stride=neck_geom(i)['stride'],
                    pad=neck_geom(i)['pad'])
    # the gate: BN + ReLU of both towers' out5 and the sigmoid aggregation, [C][Ny][Nx]
    mono_key = 'mono_layers' if dual else 'model'
    m = F.relu(folded_bn(raws['mono', 8], p, f'{mono_key}.5.bn'))[..., 0].transpose(-1, -2)
    if dual:
        s = F.relu(folded_bn(raws['stereo', 8], p, 'stereo_layers.5.bn'))[..., 0] \
            .transpose(-1, -2)
        wgt = F.conv2d(torch.cat([m, s], 1), p['aggregate_layer.weight']).sigmoid()
        ref = wgt * m + (1 - wgt) * s
    else:
        ref = m
    ck.elementwise('gate', bev, ref, cls='neck_gate_kernel')
    ck.report(report)
    return ck, report


# every z-mode / group-shape class the shipped necks launch at 220 x 300 x 12
WAYMO_CLASSES = {
    'waymo_imvoxel': ('conv_tc_neck<64->64,s1,g32,src>', 'conv_tc_neck<64->128,z2,g32,src>',
                      'conv_tc_neck<128->128,s1,g32,src>', 'conv_tc_neck<128->256,z2,g32,src>',
                      'conv_tc_neck<256->256,s1,g32,src>', 'conv_tc_neck<256->256,p0,g16,src>'),
}
WAYMO_CLASSES['waymo_dfm'] = WAYMO_CLASSES['waymo_imvoxel'] + ('conv_tc_neck<128->128,z2,g32,src>',)


@pytest.mark.gpu
@pytest.mark.parametrize('name', NECK_CASES)
def test_neck_layers_vs_fp64(name):
    ck, _ = run_neck_case(name)
    assert not ck.failures, ck.failures
    if name in WAYMO_CLASSES:
        missing = [c for c in WAYMO_CLASSES[name] if c not in ck.checked]
        assert not missing, (missing, sorted(ck.checked))


@pytest.mark.gpu
@pytest.mark.parametrize('tpi', ['2', '5'])
@pytest.mark.parametrize('name', ['neck_dfm_mt', 'neck_imvoxel_mt'])
def test_neck_multitile_items_layers(name, tpi, monkeypatch):
    """DFM_NECK_TPI is read on every launch: several tiles share one item's weight image."""
    monkeypatch.setenv('DFM_NECK_TPI', tpi)
    ck, _ = run_neck_case(name)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['neck_dfm', 'neck_imvoxel_mt'])
def test_neck_layers_simt(name):
    ck, report = run_neck_case(name, impl='simt')
    assert not any(k.startswith('conv_tc') for k in report), sorted(report)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_neck_debug_hook_refuses():
    """No stereo tower in OutdoorImVoxelNeck, no tenth layer, and the exact size only."""
    mod, x, _ = make_neck_case('neck_imvoxel')
    with torch.no_grad():
        mod(x)
    with pytest.raises(RuntimeError, match='not written'):
        mod.debug_tensor('stereo.0', (6, 5, 12, 64))
    with pytest.raises(RuntimeError, match='unknown tensor'):
        mod.debug_tensor('mono.9', (6, 5, 12, 64))
    with pytest.raises(RuntimeError, match='elements'):
        mod.debug_tensor('mono.0', (6, 5, 12, 32))
    assert mod.debug_tensor('mono.8', (6, 5, 1, 256)).abs().max() > 0


# ---------------------------------------------------------------------------------------------
# FrustumToVoxel (csrc/frustum_api.inc)
# ---------------------------------------------------------------------------------------------
FRUSTUM_CASES = {
    # tests/golden/frustum.npz's inputs: 24 x 20 x 8 voxels
    'frustum': dict(fixture=True),
    # two convs: conv1 reads GN + ReLU of conv0 from the double buffer
    'frustum_two_convs': dict(seed=41, h=64, w=160, d=12, n_voxels=(40, 36, 12), num_3dconvs=2),
    # the KITTI grid, 20 x 304 x 288 voxels: conv0 on the windowed K-outer kernel (conv_tck)
    'frustum_kitti': dict(seed=51, h=384, w=1248, d=112, n_voxels=(288, 304, 20)),
}


def make_frustum(name, impl='auto'):
    from depth_from_motion_b200 import modules
    from depth_from_motion_b200 import synthetic as syn
    from tests.util import load_frustum_case
    c = FRUSTUM_CASES[name]
    if c.get('fixture'):
        case, _ = load_frustum_case()
        nconv = 1
    else:
        nconv = c.get('num_3dconvs', 1)
        case = syn.make_frustum_case(c['seed'], c['h'], c['w'], c['d'], c['n_voxels'],
                                     num_3dconvs=nconv)
    m = modules.FrustumToVoxel(num_3dconvs=nconv, conv_impl=impl)
    m.load_state_dict(case['params'], strict=True)
    m = m.cuda().eval()
    m.coordinates_3d = case['coordinates_3d']
    m.depth_cfg = case['depth_cfg']
    return m, case, nconv


def frustum_gather_ref(case, dev):
    """feature_transformation.py:84-160 (oracle.frustum_to_voxel_forward before the convs) on
    the fp64 features, with the oracle's own sampling grid; plus the voxels whose sample point
    lies on an edge of a validity mask (where fp32 rounding can flip the mask)."""
    cfg = case['depth_cfg']
    _, sm, _ = O.depth_head_forward(case['cost'].double(), O.depth_samples(cfg).double(), 4)
    meta = case['metas'][0]
    norm, valid2d, valid = O.frustum_grid(case['coordinates_3d'], meta['cam2img'],
                                          meta['pad_shape'], cfg)
    g = norm[None].double().to(dev)
    voxel = F.grid_sample(case['stereo'].double().to(dev), g, align_corners=True)
    voxel = voxel * valid.double().to(dev)[None, None]
    disp = F.grid_sample(sm.to(dev), g, align_corners=True) * valid.double().to(dev)[None, None]
    g2 = g.clone()
    g2[..., 2] = 0
    v2 = F.grid_sample(case['sem'].double().to(dev).unsqueeze(2), g2, align_corners=True)
    v2 = v2 * valid2d.double().to(dev)[None, None] * disp
    # mask edges: within 1e-5 (normalised) of the image border or the depth range
    ph, pw = meta['pad_shape'][:2]
    px = (norm[..., 0] + 1) / 2 * (pw - 1)
    py = (norm[..., 1] + 1) / 2 * (ph - 1)
    eps = 1e-5
    edge = ((px.abs() < eps * pw) | ((px - pw).abs() < eps * pw) | (py.abs() < eps * ph) |
            ((py - ph).abs() < eps * ph) | ((norm[..., 2].abs() - 1).abs() < eps))
    return torch.cat([voxel, v2], 1), edge.to(dev)


def _gn(x, p, prefix):
    return F.group_norm(x, 32, p[prefix + '.weight'], p[prefix + '.bias'], O.GN_EPS)


def run_frustum_case(name, impl='auto'):
    from depth_from_motion_b200 import modules
    m, case, nconv = make_frustum(name, impl)
    nz, ny, nx = case['coordinates_3d'].shape[:3]
    stereo, cost, sem = case['stereo'].cuda(), case['cost'].cuda(), case['sem'].cuda()
    out, report = profiled(lambda: m(stereo, modules.CostLogits(cost), case['metas'], sem))
    p = fp64(case['params'], 'cuda')
    ck = Checker(name + ('' if impl == 'auto' else f' [{impl}]'))
    vox = _cl(m.debug_tensor('vox', (nz, ny, nx, 64)))
    ref, edge = frustum_gather_ref(case, 'cuda')
    keep = ~edge
    assert bool(keep.any())
    ck.elementwise('gather', vox[..., keep], ref[..., keep], tol=GATHER_TOL,
                   cls='frustum_gather', excluded=int(edge.sum()))
    x = vox
    raw = None
    for i in range(nconv):
        if i:
            x = F.relu(_gn(raw, p, f'voxel_convs.{i - 1}.0.gn'))
        raw = _cl(m.debug_tensor(f'conv{i}', (nz, ny, nx, 32)))
        cin = x.shape[1]
        dims = (nz, ny, nx)
        cls = classes_of(report, ('conv_tc', 'conv_tck', 'conv_simt'), cin, 32, ('s1',), dims)
        tck = any(c.startswith('conv_tck') for c in cls)
        # the windowed K-outer kernel tiles H x W by 16 x 8 and cuts D into windows of
        # neck_dhw_plan's length; the resident-weight kernel tiles W x H by 8 x 16
        ztile = 4 if tck else 0
        ck.conv(f'conv{i}', raw, x, p[f'voxel_convs.{i}.0.conv.weight'], cls, LC.k_of(cin),
                tiles=(ztile, 16, 8), simt=impl == 'simt')
    if nconv >= 3:
        with pytest.raises(RuntimeError, match='not written'):
            m.debug_tensor('conv0', (nz, ny, nx, 32))
    pooled = F.avg_pool3d(F.relu(_gn(raw, p, f'voxel_convs.{nconv - 1}.0.gn')), (4, 1, 1))
    ck.elementwise('gn+relu+pool', out, pooled, cls='frustum_pool')
    ck.report(report)
    return ck, report


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(FRUSTUM_CASES))
def test_frustum_layers_vs_fp64(name):
    ck, _ = run_frustum_case(name)
    assert not ck.failures, ck.failures
    if name == 'frustum_kitti' and not os.environ.get('DFM_NO_NTK'):
        assert 'conv_tck<64->32,s1,src>' in ck.checked, sorted(ck.checked)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['frustum', 'frustum_two_convs'])
def test_frustum_layers_simt(name):
    ck, report = run_frustum_case(name, impl='simt')
    assert not any(k.startswith('conv_tc') for k in report), sorted(report)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_frustum_debug_hook_refuses():
    """A conv beyond num_3dconvs was not written; a wrong size is refused."""
    from depth_from_motion_b200 import modules
    m, case, _ = make_frustum('frustum')
    nz, ny, nx = case['coordinates_3d'].shape[:3]
    with torch.no_grad():
        m(case['stereo'].cuda(), modules.CostLogits(case['cost'].cuda()), case['metas'],
          case['sem'].cuda())
    with pytest.raises(RuntimeError, match='not written'):
        m.debug_tensor('conv1', (nz, ny, nx, 32))
    with pytest.raises(RuntimeError, match='elements'):
        m.debug_tensor('vox', (nz, ny, nx, 32))


# ---------------------------------------------------------------------------------------------
# BEVHourglass + LIGAAnchor3DHead (csrc/bev_api.inc)
# ---------------------------------------------------------------------------------------------
BEV_CASES = {'bev': dict(seed=91, nz=5, ny=44, nx=36),          # the bev_stage.npz inputs
             'bev_kitti': dict(seed=93, nz=5, ny=304, nx=288)}  # the KITTI BEV grid
BEV_TILE = (16, 8)   # conv_tc_neck as an Nz = 1 conv over [Ny][Nx]: 16 along Ny, 8 along Nx
HG = 'bev_hourglass.'


def make_bev(name, impl='auto'):
    from depth_from_motion_b200 import modules
    from depth_from_motion_b200 import synthetic as syn
    c = syn.make_bev_case(**BEV_CASES[name])
    gn = dict(type='GN', num_groups=32, requires_grad=True)
    bev = modules.BEVHourglass(c['volume'].shape[1] * c['volume'].shape[2], 64, norm_cfg=gn,
                               conv_impl=impl)
    bev.load_state_dict(c['bev'], strict=True)
    head = modules.LIGAAnchor3DHead(
        num_classes=3, in_channels=64, feat_channels=64, num_convs=2, norm_cfg=gn,
        use_direction_classifier=True,
        anchor_generator=dict(type='Anchor3DRangeGenerator',
                              ranges=[[2, -30.4, -1.78, 59.6, 30.4, -1.78]] * 3,
                              sizes=[[3.9, 1.6, 1.56], [0.8, 0.6, 1.73], [1.76, 0.6, 1.73]],
                              rotations=[0, 1.57]), conv_impl=impl)
    head.load_state_dict(c['head'], strict=True)
    return bev.cuda().eval(), head.cuda().eval(), c


def run_bev_case(name, impl='auto'):
    bev, head, c = make_bev(name, impl)
    v = c['volume'].cuda()
    x = v.view(1, -1, v.shape[3], v.shape[4])

    def fwd():
        pre, feat = bev(x)
        return pre, feat, head.forward_single(feat)
    (prehg, feat, (cls, box, dirc)), report = profiled(fwd)
    h, w = x.shape[2:]
    pb, ph = fp64(c['bev'], 'cuda'), fp64(c['head'], 'cuda')
    simt = impl == 'simt'
    ck = Checker(name + ('' if simt is False else ' [simt]'))

    def layer(mod, label, cin, cout, stride, transposed, hw, xin, wt):
        raw = _cl(mod.debug_tensor(label, hw + (cout,)))
        mode = 'T' if transposed else ('s2' if stride == 2 else 's1')
        cls = classes_of(report, ('conv2d_tc',), cin, cout, (mode,), hw + (1,))
        cls += classes_of(report, ('conv2d_simt',), cin, cout, (mode,), (1,) + hw)
        tc = any(k.startswith('conv2d_tc') for k in cls)
        ck.conv(f'{label}', raw, xin, wt, cls, LC.k_of(cin, transposed, nd=2),
                tiles=BEV_TILE if tc else (0, 0), simt=simt or not tc, stride=stride,
                transposed=transposed)
        return raw
    xd = x.double()
    h2, w2, h4, w4 = h // 2, w // 2, h // 4, w // 4
    r0 = layer(bev, 'compress', x.shape[1], 64, 1, False, (h, w), xd,
               pb['compress_conv.conv.weight'])
    a0 = F.relu(_gn(r0, pb, 'compress_conv.gn'))
    r1 = layer(bev, 'conv1', 64, 128, 2, False, (h2, w2), a0, pb[HG + 'conv1.0.0.weight'])
    r2 = layer(bev, 'conv2', 128, 128, 1, False, (h2, w2), F.relu(_gn(r1, pb, HG + 'conv1.0.1')),
               pb[HG + 'conv2.0.weight'])
    pre = F.relu(_gn(r2, pb, HG + 'conv2.1'))
    r3 = layer(bev, 'conv3', 128, 128, 2, False, (h4, w4), pre, pb[HG + 'conv3.0.0.weight'])
    r4 = layer(bev, 'conv4', 128, 128, 1, False, (h4, w4), F.relu(_gn(r3, pb, HG + 'conv3.0.1')),
               pb[HG + 'conv4.0.0.weight'])
    r5 = layer(bev, 'conv5', 128, 128, 1, True, (h2, w2), F.relu(_gn(r4, pb, HG + 'conv4.0.1')),
               pb[HG + 'conv5.0.weight'])
    post = F.relu(_gn(r5, pb, HG + 'conv5.1') + pre)
    r6 = layer(bev, 'conv6', 128, 64, 1, True, (h, w), post, pb[HG + 'conv6.0.weight'])
    ck.elementwise('prehg emit', prehg, a0, cls='bev_emit')
    ck.elementwise('out emit', feat, _gn(r6, pb, HG + 'conv6.1'), cls='bev_emit')
    # the head on the GPU's own BEV features
    xf = feat.double()
    srcs = {'cls': xf, 'reg': xf}
    for i in range(2):
        for br in ('cls', 'reg'):
            r = layer(head, f'{br}{i}', 64, 64, 1, False, (h, w), srcs[br],
                      ph[f'{br}_convs.{i}.conv.weight'])
            srcs[br] = F.relu(_gn(r, ph, f'{br}_convs.{i}.gn'))
    # the output convs at their padded widths: conv_cls rows 0..17, the 1x1 conv_dir_cls in the
    # centre tap of rows 18..29, zero rows up to 32; conv_reg rows 0..41, zero rows up to 64
    wc = torch.zeros(32, 64, 3, 3, dtype=torch.float64, device='cuda')
    wc[:18] = ph['conv_cls.weight']
    wc[18:30, :, 1, 1] = ph['conv_dir_cls.weight'][:, :, 0, 0]
    wr = torch.zeros(64, 64, 3, 3, dtype=torch.float64, device='cuda')
    wr[:42] = ph['conv_reg.weight']
    rc = layer(head, 'cls_out', 64, 32, 1, False, (h, w), srcs['cls'], wc)
    rr = layer(head, 'reg_out', 64, 64, 1, False, (h, w), srcs['reg'], wr)
    if not (torch.all(rc[:, 30:] == 0) and torch.all(rr[:, 42:] == 0)):
        ck.failures.append(('padded output columns are not exactly 0',
                            float(rc[:, 30:].abs().max()), float(rr[:, 42:].abs().max())))
    ck.elementwise('cls emit', cls, rc[:, :18] + ph['conv_cls.bias'][:, None, None],
                   cls='bev_emit')
    ck.elementwise('dir emit', dirc, rc[:, 18:30] + ph['conv_dir_cls.bias'][:, None, None],
                   cls='bev_emit')
    ck.elementwise('reg emit', box, rr[:, :42] + ph['conv_reg.bias'][:, None, None],
                   cls='bev_emit')
    ck.report(report)
    return ck, report


# the shipped 304 x 288 stage launches these classes
BEV_CLASSES = ('conv2d_tc<160->64,s1,g16,src>', 'conv2d_tc<128->128,s1,g16,src>',
               'conv2d_tc<64->64,s1,g16,src>', 'conv2d_tc<64->32,s1,g32,src>',
               'conv2d_simt<64->128,s2,src>', 'conv2d_simt<128->128,s2,src>',
               'conv2d_simt<128->128,T,src>', 'conv2d_simt<128->64,T,src>')


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(BEV_CASES))
def test_bev_stage_layers_vs_fp64(name):
    ck, _ = run_bev_case(name)
    assert not ck.failures, ck.failures
    if name == 'bev_kitti':
        missing = [c for c in BEV_CLASSES if c not in ck.checked]
        assert not missing, (missing, sorted(ck.checked))


@pytest.mark.gpu
def test_bev_stage_layers_simt():
    ck, report = run_bev_case('bev', impl='simt')
    assert not any(k.startswith('conv2d_tc') for k in report), sorted(report)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_bev_debug_hooks_refuse():
    bev, head, c = make_bev('bev')
    v = c['volume'].cuda()
    with torch.no_grad():
        head.forward_single(bev(v.view(1, -1, v.shape[3], v.shape[4]))[1])
    with pytest.raises(RuntimeError, match='not written'):
        head.debug_tensor('cls2', (44, 36, 64))
    with pytest.raises(RuntimeError, match='elements'):
        head.debug_tensor('reg_out', (44, 36, 42))
    with pytest.raises(RuntimeError, match='unknown tensor'):
        bev.debug_tensor('conv7', (44, 36, 64))


# ---------------------------------------------------------------------------------------------
# A/B switch arms: each is read once per process, so each runs in its own interpreter
# ---------------------------------------------------------------------------------------------
AB_ARMS = [
    # (env, test, a class the arm must launch, a default-path class it must not launch)
    ({'DFM_NECK_CG32': '1'}, 'test_neck_layers_vs_fp64 and neck_dfm_mt',
     'conv_tc_neck<256->256,p0,g32,src>', ',g16,'),
    ({'DFM_NECK_WIN': '1'}, 'test_neck_layers_vs_fp64 and neck_imvoxel_mt',
     'conv_tc_neck<64->64,s1,g16,src>', 'conv_tc_neck<64->64,s1,g32,src>'),
    ({'DFM_NO_NTK': '1'}, 'test_frustum_layers_vs_fp64 and frustum_kitti',
     'conv_tc<64->32,s1,src>', 'conv_tck'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('arm', AB_ARMS, ids=lambda a: ','.join(f'{k}={v}' for k, v in a[0].items()))
def test_ab_arm_stage_layers(arm):
    env_add, sel, want, avoid = arm
    env = dict(os.environ, **env_add)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-s',
                        '-m', 'gpu', '-p', 'no:cacheprovider', '-k', sel],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    print(out[-6000:])
    classes = [ln for ln in out.splitlines() if ln.startswith('CLASSES')]
    assert r.returncode == 0, out[-6000:]
    assert classes, out[-2000:]
    assert want in classes[0], classes[0]
    assert avoid not in classes[0], classes[0]


# ---------------------------------------------------------------------------------------------
# CPU: the bounds keep a lost product term out, for every new layer class
# ---------------------------------------------------------------------------------------------
def _cpu_neck_rows():
    from depth_from_motion_b200 import modules
    from depth_from_motion_b200 import synthetic as syn
    from tests.util import make_neck_mt_case
    rows = []
    rng, x = make_neck_mt_case('neck_dfm_mt')
    sd = syn.make_neck_params(rng, modules.DfMNeck(64, 256, num_frames=2).state_dict())
    p = fp64(sd, 'cpu')
    x = x.double()
    for tower, xin in (('stereo_layers', x), ('mono_layers', x[:, :64])):
        out = {}
        for i, xi in neck_layers(xin, p, tower, out.__getitem__):
            w = p[f'{tower}.{NECK_KEYS[i]}.conv.weight']
            g = neck_geom(i)
            out[i] = LC.conv_planes(xi, w, **g)
            rows.append((f'{tower}.{i} {NECK_ZMODE[i]} K={LC.k_of(xi.shape[1])}', xi, w, g,
                         out[i], LC.k_of(xi.shape[1])))
    return rows


def _cpu_bev_rows():
    from depth_from_motion_b200 import synthetic as syn
    c = syn.make_bev_case(**BEV_CASES['bev'])
    pb, ph = fp64(c['bev'], 'cpu'), fp64(c['head'], 'cpu')
    x = c['volume'].double().flatten(1, 2)
    rows = []

    def conv(label, xi, w, stride=1, transposed=False):
        g = dict(stride=stride, transposed=transposed)
        y = LC.conv_planes(xi, w, **g)
        rows.append((label, xi, w, g, y, LC.k_of(xi.shape[1], transposed, nd=2)))
        return y
    r0 = conv('compress', x, pb['compress_conv.conv.weight'])
    a0 = F.relu(_gn(r0, pb, 'compress_conv.gn'))
    r1 = conv('conv1 s2', a0, pb[HG + 'conv1.0.0.weight'], 2)
    r2 = conv('conv2', F.relu(_gn(r1, pb, HG + 'conv1.0.1')), pb[HG + 'conv2.0.weight'])
    pre = F.relu(_gn(r2, pb, HG + 'conv2.1'))
    r3 = conv('conv3 s2', pre, pb[HG + 'conv3.0.0.weight'], 2)
    r4 = conv('conv4', F.relu(_gn(r3, pb, HG + 'conv3.0.1')), pb[HG + 'conv4.0.0.weight'])
    r5 = conv('conv5 T', F.relu(_gn(r4, pb, HG + 'conv4.0.1')), pb[HG + 'conv5.0.weight'],
              transposed=True)
    r6 = conv('conv6 T', F.relu(_gn(r5, pb, HG + 'conv5.1') + pre), pb[HG + 'conv6.0.weight'],
              transposed=True)
    feat = _gn(r6, pb, HG + 'conv6.1')
    r = conv('head cls0', feat, ph['cls_convs.0.conv.weight'])
    r = conv('head cls1', F.relu(_gn(r, ph, 'cls_convs.0.gn')), ph['cls_convs.1.conv.weight'])
    wc = torch.zeros(32, 64, 3, 3, dtype=torch.float64)
    wc[:18] = ph['conv_cls.weight']
    wc[18:30, :, 1, 1] = ph['conv_dir_cls.weight'][:, :, 0, 0]
    conv('head cls_out', F.relu(_gn(r, ph, 'cls_convs.1.gn')), wc)
    r = conv('head reg0', feat, ph['reg_convs.0.conv.weight'])
    r = conv('head reg1', F.relu(_gn(r, ph, 'reg_convs.0.gn')), ph['reg_convs.1.conv.weight'])
    wr = torch.zeros(64, 64, 3, 3, dtype=torch.float64)
    wr[:42] = ph['conv_reg.weight']
    conv('head reg_out', F.relu(_gn(r, ph, 'reg_convs.1.gn')), wr)
    return rows


def _cpu_frustum_rows():
    from tests.util import load_frustum_case
    case, _ = load_frustum_case()
    vox, _ = frustum_gather_ref(case, 'cpu')
    p = fp64(case['params'], 'cpu')
    w = p['voxel_convs.0.0.conv.weight']
    return [('frustum conv0', vox, w, {}, LC.conv_planes(vox, w), LC.k_of(64))]


@pytest.mark.parametrize('stage', ['neck', 'frustum', 'bev'])
def test_stage_bounds_separate_lost_term(stage):
    """On oracle fp64 inputs at the fixture shapes, for every conv class of the stage (the neck
    up to K = 27 * 256 = 6912): the tensor-core bound max(K_E3 e3, floor) and the fp32 floor
    of the CUDA-core kernels both stay SEPARATION times below e2, in the normalised max-norm and
    element-wise (error over the product scale)."""
    torch.set_num_threads(max(1, os.cpu_count() or 8))
    with torch.no_grad():
        rows = dict(neck=_cpu_neck_rows, frustum=_cpu_frustum_rows, bev=_cpu_bev_rows)[stage]()
        res = []
        for label, x, w, g, ref, k in rows:
            ys = LC.emulated_outputs(x, w, **g)
            e3, e2 = LC.norm_errors(ys, ref)
            _, el3, el2, elb = elementwise_errors(ref, ref, *ys, LC.product_scale(x, w, **g), k,
                                                  FLOOR_C)
            res.append((label, k, e3, e2, layer_bound(e3, k, FLOOR_C), el3, el2, elb))
    print(f'\n{stage}: layer | e3 | e2 | bound | e2 / bound | e2 / floor || element-wise: '
          f'e3 | e2 | bound | e2 / bound')
    for label, k, e3, e2, b, el3, el2, elb in res:
        print(f'  {label:34s} {e3:.2e} {e2:.2e} {b:.2e} {e2 / b:6.1f} '
              f'{e2 / LC.acc_floor(k, FLOOR_C):6.1f}'
              f' || {el3:.2e} {el2:.2e} {elb:.2e} {el2 / elb:6.1f}')
    assert stage != 'neck' or any(r[5] == 6912 for r in rows)
    for label, k, e3, e2, b, el3, el2, elb in res:
        assert e3 > 0 and e2 > 0 and el3 > 0, label
        assert SEPARATION * b <= e2, (label, e3, e2, b)
        assert SEPARATION * LC.acc_floor(k, FLOOR_C) <= e2, (label, 'floor', e2)
        assert SEPARATION * elb <= el2, (label, 'element-wise', el3, el2, elb)


def test_conv_planes_matches_torch():
    """The shared fp64 reference conv (per-axis stride / pad, regions, 2-D and 3-D, transposed)
    equals torch's convs."""
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, 8, 7, 6, 12, generator=g, dtype=torch.float64)
    w = torch.randn(4, 8, 3, 3, 3, generator=g, dtype=torch.float64)
    for stride, pad in ((1, 1), ((1, 1, 2), 1), (1, (1, 1, 0)), (2, 1)):
        full = F.conv3d(x, w, None, stride, pad)
        assert torch.allclose(LC.conv_planes(x, w, stride=stride, pad=pad), full, atol=1e-12)
        r = ((1, 3), (0, 2), None)
        got = LC.conv_planes(x, w, stride=stride, pad=pad, region=r)
        assert torch.allclose(got, full[:, :, 1:3, 0:2], atol=1e-12), (stride, pad)
        ys = LC.emulated_outputs(x, w, stride=stride, pad=pad, region=r)
        assert torch.allclose(ys[0], got, rtol=1e-4, atol=1e-4), (stride, pad)
    x2 = x[:, :, 0]
    w2 = w[:, :, 0]
    for stride in (1, 2):
        assert torch.allclose(LC.conv_planes(x2, w2, stride=stride),
                              F.conv2d(x2, w2, None, stride, 1), atol=1e-12)
    wt = torch.randn(8, 4, 3, 3, generator=g, dtype=torch.float64)
    assert torch.allclose(LC.conv_planes(x2, wt, transposed=True),
                          F.conv_transpose2d(x2, wt, None, 2, 1, 1), atol=1e-12)
    assert math.isclose(LC.k_of(256), 6912)
