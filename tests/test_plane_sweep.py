"""The plane-sweep cost volume, element by element, against an fp64 referee.

The warp (``warp_coord`` + ``bilinear_taps`` in csrc/common.cuh, metadata from
``make_warp_geom``) builds the first tensor of the KITTI 3-D path and runs in three places: the
standalone op ``dfm_op_build_cost_volume``, the tensor-core warp loader of dres0
(``WarpLoader8``) and the SIMT ``WarpLoader``.  Every prev-half element is held to the bound of
``tests/plane_sweep_check.py`` (coordinate error derived from the fp32 evaluation order times
the local tap differences, plus a few ulps of the tap sum); the cur half must be the stride
lattice bit for bit.  Features are relu(white noise), so a coordinate error is not damped.

CPU: the referee is pinned to the reference's own ``build_dfm_cost`` in fp64, the coordinate
bound's constant is calibrated by emulating ``warp_coord`` in fp32, and planted defects of the
coordinate chain are shown to exceed the bound by SEPARATION.
GPU: the standalone op at every geometry case, dres0 under both loaders, the channels-last
entry, and DepthHead at its edge shapes.
"""
import os
import time

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import synthetic as syn
from oracle import dfm_oracle as O
from tests import layer_check as LC
from tests import plane_sweep_check as PS
from tests.layer_check import SEPARATION

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'plane_sweep_fp64.npz')

D112 = O.downsampled_depth(syn.depth_cfg_for(112))   # shipped planes: 2.257 .. 59.34 m
P2, C2P = syn.KITTI_P2, syn.KITTI_CUR2PREV[2]
P320 = syn.kitti_p2_for_width(320)

# name -> feature size, channels, planes, geometry, and the geometry each case must contain
CASES = {
    'shipped_plain': dict(h=384, w=1248, c=32, depths=D112, geom=PS.Geom(P2, C2P, (370, 1224))),
    'shipped_aug': dict(h=384, w=1248, c=32, depths=D112,
                        geom=PS.Geom(P2, C2P, (375, 1242), True, (10, 40), 1.03),
                        expect=('flip_crop_scale',)),
    # the previous camera 1.5 m ahead: near planes magnify out of the map
    'longitudinal': dict(h=96, w=320, c=16, depths=D112[:24],
                         geom=PS.Geom(P320, syn.cur2prev_pose(t=(0, 0, -1.5)), (96, 320)),
                         expect=('edge_band',)),
    'lateral': dict(h=96, w=320, c=16, depths=D112[:24],
                    geom=PS.Geom(P320, syn.cur2prev_pose(t=(2.5, 0, 0.3)), (96, 320)),
                    expect=('edge_band',)),
    # 75 deg of yaw and 11 of pitch: the plane c = 0 crosses the volume, points behind the
    # previous camera project (mirrored) onto the map
    'yaw_pitch': dict(h=96, w=320, c=16, depths=D112[::4],
                      geom=PS.Geom(P320, syn.cur2prev_pose(1.3, 0.2, (0, 0, -3.0)), (96, 320)),
                      expect=('behind_on_map', 'near_singular')),
    'identity_pose': dict(h=384, w=1248, c=8, depths=D112, geom=PS.Geom(P2, np.eye(4), (370, 1224)),
                          expect=('identity',)),
    # round(h / 4) half-even ties: 24.5 -> 24, 79.5 -> 80; 25.5 -> 26, 78.5 -> 78
    'tie_98x318': dict(h=98, w=318, c=16, depths=D112[:16], geom=PS.Geom(P320, C2P, (98, 318)),
                       expect=('tie',)),
    'tie_102x314': dict(h=102, w=314, c=16, depths=D112[:16], geom=PS.Geom(P320, C2P, (102, 314)),
                        expect=('tie',)),
    'odd_97x313': dict(h=97, w=313, c=16, depths=D112[:16], geom=PS.Geom(P320, C2P, (97, 313))),
    # KITTI P2 as the 3 x 4 calibration (translation column) instead of the padded 4 x 4
    'cam_3x4': dict(h=96, w=320, c=16, depths=D112[:16], geom=PS.Geom(P320[:3], C2P, (96, 320)),
                    expect=('cam_3x4',)),
    'near_planes': dict(h=96, w=320, c=16, depths=torch.linspace(0.5, 2.2, 16),
                        geom=PS.Geom(P320, C2P, (96, 320)), expect=('near_planes',)),
}
# the cases the fp64 pin and the CPU separation / calibration run at (shipped size, small C)
PIN_CASES = ('shipped_aug', 'yaw_pitch', 'cam_3x4')


def case_inputs(name, c=None, seed=None):
    spec = CASES[name]
    cur, prev = syn.white_noise_pair(seed if seed is not None else 1000 + list(CASES).index(name),
                                     c or spec['c'], spec['h'], spec['w'])
    return cur, prev, spec['depths'].float(), spec['geom']


def small(name):
    """The case's geometry on a 32 x 64 map (the pin fixture's size)."""
    spec = CASES[name]
    return spec['geom'], spec['depths'][::max(1, len(spec['depths']) // 8)][:8].float()


@pytest.fixture
def fp64_default():
    with PS.float64_default():
        yield


# ---------------------------------------------------------------------------------------------
# CPU: the referee
# ---------------------------------------------------------------------------------------------
def test_float64_default_is_scoped(fp64_default):
    assert torch.get_default_dtype() == torch.float64
    assert torch.linspace(0, 1, 3).dtype == torch.float64


def test_float64_default_restored():
    assert torch.get_default_dtype() == torch.float32
    with pytest.raises(RuntimeError):
        with PS.float64_default():
            raise RuntimeError('restored on the way out')
    assert torch.get_default_dtype() == torch.float32


@pytest.mark.parametrize('name', PIN_CASES)
def test_referee_pinned_to_reference_fp64(name):
    """oracle.build_dfm_cost in fp64 equals the reference's own build_dfm_cost in fp64 (stored
    by tests/golden/make_plane_sweep_golden.py; also run live when the reference tree is
    present) to 1e-12; the referee's cur half is the lattice and its prev half is the bilinear
    sample at sample_points' coordinates, both to 1e-12."""
    gold = np.load(GOLDEN)
    cur, prev = (torch.from_numpy(gold[f'{name}.{k}']) for k in ('cur', 'prev'))
    g, depths = small(name)
    vol = PS.oracle_volume(cur, prev, depths, g)
    assert vol.dtype == torch.float64 and torch.get_default_dtype() == torch.float32
    want = torch.from_numpy(gold[f'{name}.volume'])
    scale = float(want.abs().max())
    assert float((vol - want).abs().max()) <= 1e-12 * scale
    from oracle import ref_loader
    if ref_loader.reference_available():
        live = PS.oracle_volume(cur, prev, depths, g, ref_loader.load_reference().build_dfm_cost)
        assert float((vol - live).abs().max()) <= 1e-12 * scale
    c = cur.shape[1]
    ho, wo = vol.shape[-2:]
    assert float((vol[:, :c] - PS.lattice(cur.double(), 4, ho, wo)).abs().max()) <= 1e-12 * scale
    pts = PS.sample_points(g, depths, ho, wo)
    ok = ~PS.near_singular(pts)
    assert bool(ok.any())
    diff = (vol[:, c:] - PS.bilinear(prev.double(), pts['fx'], pts['fy'])).abs()
    assert float(diff[..., ok].max()) <= 1e-12 * scale


def test_delta_calibration():
    """warp_coord emulated in fp32 (both fma-contraction variants) against the fp64 sample
    points, at every case's geometry: the worst |fp32 - fp64| over the unit coordinate bound
    stays below K_DELTA / 2 and is not vacuous."""
    rows = []
    for name, spec in CASES.items():
        g, depths = spec['geom'], spec['depths'].float()
        ho, wo = PS.out_size(spec['h'], spec['w'], g.csf)
        pts = PS.sample_points(g, depths, ho, wo)
        ok = ~PS.near_singular(pts).numpy()
        worst = 0.0
        for contract in (False, True):
            fx, fy = PS.emulate_warp_coord(g, depths.numpy(), ho, wo, contract)
            for got, ref, d1 in ((fx, pts['fx'], pts['dx1']), (fy, pts['fy'], pts['dy1'])):
                r = np.abs(got.astype(np.float64) - ref.numpy()) / d1.numpy()
                assert np.isfinite(r[ok]).all(), name
                worst = max(worst, float(r[ok].max()))
        rows.append((name, worst))
    print('\ncase | worst |fp32 - fp64| / unit coordinate bound')
    for name, worst in rows:
        print(f'  {name:14s} {worst:.3f}')
    top = max(w for _, w in rows)
    assert 0.5 < top <= PS.K_DELTA / 2, rows


# separation shift per case and defect: 2e-3 px everywhere except x under a flip, where the fp32
# subtraction org_w - u carries rounding of org_w's size (about 3e-4 px at 1242 px) on every
# element; 3e-3 px is the smallest x shift that separates 3x there (measured ratio at 2e-3: 2.2)
SEPARATION_SHIFT = {('shipped_aug', 'shift_x'): 3e-3}


@pytest.mark.parametrize('name', ('shipped_plain', 'shipped_aug'))
def test_defects_separate(name):
    """Each planted defect of the coordinate chain, sampled in fp64, exceeds the per-element
    bound by at least SEPARATION on some element, at the shipped size (4 channels)."""
    torch.set_num_threads(max(1, os.cpu_count() or 8))
    spec = CASES[name]
    g = spec['geom']
    _, prev = syn.white_noise_pair(5, 4, spec['h'], spec['w'])
    prev = prev.double()
    ho, wo = PS.out_size(spec['h'], spec['w'], g.csf)
    pts = PS.sample_points(g, spec['depths'].float(), ho, wo)
    ref = PS.bilinear(prev, pts['fx'], pts['fy'])
    bound = PS.prev_bound(prev, pts)
    rows = []
    for defect in PS.DEFECTS:
        if defect in ('crop_after_scale', 'flip_about_w_minus_1') and not g.flip:
            continue   # no crop / scale / flip to get wrong
        shift = SEPARATION_SHIFT.get((name, defect), 2e-3)
        if defect == 'align_corners_false':
            v = PS.bilinear(prev, pts['fx'], pts['fy'], align_corners=False)
        else:
            dp = PS.sample_points(g, spec['depths'].float(), ho, wo, defect=defect, shift=shift)
            v = PS.bilinear(prev, dp['fx'], dp['fy'])
        rows.append((defect, shift, float(PS.ratio((v - ref).abs(), bound).max())))
    print(f'\n{name}: defect | shift px | worst |defect - referee| / bound')
    for defect, shift, r in rows:
        print(f'  {defect:22s} {shift:.0e} {r:10.2f}')
    assert all(r >= SEPARATION for _, _, r in rows), rows


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def geometry_proof(name, pts, depths):
    """Counts that show the case holds the geometry it names ([D, ho, wo] positions)."""
    spec = CASES[name]
    g, h, w = spec['geom'], spec['h'], spec['w']
    fx, fy, c = pts['fx'], pts['fy'], pts['c']
    on_map = (fx > -1) & (fx < w) & (fy > -1) & (fy < h)
    band = on_map & ((fx < 0) | (fx > w - 1) | (fy < 0) | (fy > h - 1))
    return dict(edge_band=int(band.sum()), behind_on_map=int(((c < 0) & on_map).sum()),
                near_singular=int(PS.near_singular(pts).sum()),
                flip_crop_scale=int(g.flip and g.crop != (0, 0) and g.scale != 1.0),
                identity=int(np.array_equal(g.cur2prev, np.eye(4))),
                tie=int(any(abs(n / 4 - round(n / 4)) == 0.5 for n in (h, w))),
                cam_3x4=int(g.cam2img.shape == (3, 4)),
                near_planes=int(float(depths.min()) < float(D112.min())))


def gpu_volume(cur, prev, depths, g):
    from depth_from_motion_b200 import modules
    return modules.build_dfm_cost(cur.cuda(), prev.cuda(), depths, g.fsf, g.csf,
                                  torch.as_tensor(g.cam2img[None]), g.cur2prev[None],
                                  g.ori_shape, g.flip, g.crop, img_scale_factor=g.scale)


def check_prev_half(got, ref, prev, pts):
    """(worst err / bound over regular elements, near-singular positions, positions of those
    where GPU and referee are not both 0 and differ by more than 4 ulps of the tap scale)."""
    bound = PS.prev_bound(prev, pts)
    err = (got - ref).abs()
    ns = PS.near_singular(pts)
    r = torch.where(ns[None, None], torch.zeros_like(err), PS.ratio(err, bound))
    worst = float(r.max())
    k, z, y, x = np.unravel_index(int(torch.argmax(r.reshape(-1))), r.shape[1:])
    where = dict(k=k, z=z, y=y, x=x, fx=float(pts['fx'][z, y, x]), fy=float(pts['fy'][z, y, x]),
                 got=float(got[0, k, z, y, x]), ref=float(ref[0, k, z, y, x]),
                 bound=float(bound[0, k, z, y, x]))
    tiny = PS.EPS_V_ULPS * PS.U32 * float(prev.abs().max())
    odd = ns & (err > tiny).any(1)[0]
    return worst, int(ns.sum()), int(odd.sum()), where


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_cost_volume_op(name):
    """dfm_op_build_cost_volume over the whole volume: cur half == lattice bit for bit, every
    prev element within the bound; near-singular elements agree or are counted (few)."""
    t0 = time.time()
    spec = CASES[name]
    cur, prev, depths, g = case_inputs(name)
    with torch.no_grad():
        vol = gpu_volume(cur, prev, depths, g).double()
        cur_d, prev_d = cur.cuda().double(), prev.cuda().double()
        ref = PS.referee(cur_d, prev_d, depths, g)
    c = cur.shape[1]
    d, ho, wo = ref.shape[2:]
    assert vol.shape == ref.shape
    assert torch.equal(vol[:, :c], PS.lattice(cur_d, g.csf, ho, wo).expand(-1, -1, d, -1, -1))
    pts = PS.sample_points(g, depths, ho, wo, 'cuda')
    worst, n_ns, n_odd, where = check_prev_half(vol[:, c:], ref[:, c:], prev_d, pts)
    proof = geometry_proof(name, pts, depths)
    on_map_behind = (pts['c'] < 0) & (vol[0, c:] != 0).any(0)
    proof['behind_sampled'] = int(on_map_behind.sum())
    print(f'\n{name} [{c}x{d}x{ho}x{wo}]: worst err/bound {worst:.3f}, near-singular {n_ns}, '
          f'unexplained-by-bound {n_odd}, geometry {proof}, {time.time() - t0:.1f} s')
    assert worst <= 1.0, (name, worst, where)
    assert n_odd <= max(8, 1e-3 * d * ho * wo), (name, n_odd)
    for tag in spec.get('expect', ()):
        assert proof[tag] > 0, (name, tag, proof)
    if 'behind_on_map' in spec.get('expect', ()):
        assert proof['behind_sampled'] > 0, proof   # mirrored samples are not zeroed


# dres0 of the stereo tower, both loaders: three geometries at 96 x 320
DRES0_CASES = ('lateral', 'yaw_pitch', 'cam_3x4')


def dres0_check(name, impl, c_twin=False):
    """raw0 of DfMBackbone(conv_impl=impl) against the fp64 conv of the referee's volume:
    |gpu - ref| <= layer_bound * sum |x| |w| + conv(|w|, warp bound of each input)."""
    from depth_from_motion_b200 import modules
    spec = CASES[name]
    cur, prev, depths, g = case_inputs(name, c=32)
    params = syn.make_backbone_params(np.random.RandomState(7), len(depths))
    cfg = syn.depth_cfg_for(len(depths))
    m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg, conv_impl=impl).cuda().eval()
    m.load_state_dict(params, strict=True)
    m.downsampled_depth = depths
    with torch.no_grad():
        m(cur.cuda(), prev.cuda(), [g.meta()])
        ho, wo = PS.out_size(spec['h'], spec['w'], 4)
        d = len(depths)
        got = m.debug_tensor('raw0', (d, ho, wo, 32)).permute(3, 0, 1, 2)[None].double()
        cur_d, prev_d = cur.cuda().double(), prev.cuda().double()
        ref_vol = PS.referee(cur_d, prev_d, depths, g)
        pts = PS.sample_points(g, depths, ho, wo, 'cuda')
        bvol = PS.warp_input_bound(prev_d, ref_vol[:, 32:], pts, 32)
        w = params['dres0.conv.weight'].cuda().double()
        geo = dict(stride=1, region=((0, d), None, None))
        ref = LC.conv_planes(ref_vol, w, **geo)
        y3, _, _ = LC.emulated_outputs(ref_vol, w, **geo)
        scale = LC.product_scale(ref_vol, w, **geo)
        slack = LC.conv_planes(bvol, w.abs(), **geo)
    s = scale.clamp_min(1e-12 * float(scale.max()))
    k = LC.k_of(64)
    elb = LC.layer_bound(float(((y3 - ref).abs() / s).max()), k)
    r = float(((got - ref).abs() / (elb * s + slack)).max())
    warp_share = float((slack / (elb * s + slack)).max())
    m.release()
    return r, warp_share


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ('auto', 'simt'))
@pytest.mark.parametrize('name', DRES0_CASES)
def test_dres0_warp_loader(name, impl):
    """dres0's loaders (auto: tensor-core WarpLoader8, simt: WarpLoader) against the fp64 conv
    of the referee's volume, element-wise."""
    r, share = dres0_check(name, impl)
    print(f'\ndres0 {impl} {name}: worst err/bound {r:.3f} (largest warp share of a bound '
          f'{share:.2f})')
    assert r <= 1.0, (name, impl, r)


@pytest.mark.gpu
def test_channels_last_entry_same_bits():
    """dfm_backbone_forward_cl (stereo features with an SPPUNetNeckTail-style channels-last
    twin) gives the bits of the NCHW entry: outputs and dres0's raw output."""
    from depth_from_motion_b200 import modules
    cur, prev, depths, g = case_inputs('shipped_aug', c=32)
    params = syn.make_backbone_params(np.random.RandomState(8), len(depths))
    m = modules.DfMBackbone(in_channels=32, depth_cfg=syn.depth_cfg_for(len(depths))).cuda().eval()
    m.load_state_dict(params, strict=True)
    m.downsampled_depth = depths
    d, ho, wo = len(depths), 96, 312
    res = []
    with torch.no_grad():
        for twin in (False, True):
            a, b = cur.cuda(), prev.cuda()
            if twin:
                a._dfm_cl = a[0].permute(1, 2, 0).contiguous()
                b._dfm_cl = b[0].permute(1, 2, 0).contiguous()
            out = m(a, b, [g.meta()])
            res.append([t.clone() for t in out] + [m.debug_tensor('raw0', (d, ho, wo, 32))])
    m.release()
    for x, y, key in zip(*res, ('cost', 'stereo', 'mono', 'raw0')):
        assert torch.equal(x, y), key


# DepthHead edges: (D, Ho, Wo, factor, logits).  OW = Wo * f % 4 == 0 takes depth_head4, the
# rest the one-pixel kernel; Ho, Wo of 1 or 2 hit the OW > 1 / OH > 1 branches; D = 112 is the
# shipped 448 bins, where the empty-interval fix-up of depth_head4 can fire
DH_CASES = [
    (12, 5, 8, 4, 'randn'), (12, 5, 7, 3, 'randn'), (12, 1, 1, 4, 'randn'),
    (12, 2, 1, 2, 'randn'), (12, 1, 2, 2, 'randn'), (12, 2, 2, 3, 'randn'),
    (12, 3, 6, 2, 'pm40'), (12, 3, 5, 3, 'equal'), (112, 3, 8, 4, 'randn'),
    (112, 2, 5, 4, 'pm40'), (112, 2, 3, 3, 'randn'), (112, 1, 4, 4, 'equal'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', DH_CASES, ids=lambda c: 'd{}_{}x{}_f{}_{}'.format(*c))
def test_depth_head_edges(case):
    """dfm_depth_head_forward element-wise against oracle.depth_head_forward in fp64."""
    from depth_from_motion_b200 import modules
    d, ho, wo, f, kind = case
    g = torch.Generator().manual_seed(d * 100 + ho * 10 + wo + f)
    if kind == 'randn':
        cost = torch.randn(1, 1, d, ho, wo, generator=g) * 3
    elif kind == 'pm40':
        cost = (torch.rand(1, 1, d, ho, wo, generator=g) * 2 - 1) * 40
    else:
        cost = torch.full((1, 1, d, ho, wo), 1.7)
    cfg = dict(num_bins=f * d, depth_min=2, depth_max=59.6, downsample_factor=f)
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2, max_depth=59.6),
        with_convs=False, num_views=1, depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = f
    try:
        vol, sm, preds = head(cost.cuda())
    except RuntimeError as e:
        # the one-pixel kernel stages a column of D f bins and refuses what does not fit
        assert (wo * f) % 4 != 0 and 'too many depth planes' in str(e), e
        print(f'\n{case}: rejected ({e})')
        return
    rvol, rsm, rpreds = O.depth_head_forward(cost.double(), O.depth_samples(cfg).double(), f)
    assert vol.shape == rvol.shape and sm.shape == rsm.shape and preds.shape == rpreds.shape
    cmax = float(cost.abs().max())
    # vol: the fp32 source index sz * k of the z interpolation carries about D ulps (k < D f),
    # which moves the weights by as much; plus the fp32 blends of values up to max |cost|
    b_vol = (8 + 2 * d) * PS.U32 * cmax
    e_vol = float((vol.double().cpu() - rvol).abs().max()) / b_vol
    # softmax: ex2.approx and the fp32 argument (v - max) * log2(e), and the logit error of vol
    # twice (the value and the normaliser) -- relative to each probability, plus an absolute
    # floor for probabilities that underflow; preds inherit the same relative error
    rel = 2e-5 + 2 * b_vol
    e_sm = float(((sm.double().cpu() - rsm).abs() / (rel * rsm + 1e-7)).max())
    e_pr = float((preds.double().cpu() - rpreds).abs().max()) / (rel * float(rpreds.abs().max()))
    print(f'\n{case}: err / bound  vol {e_vol:.3f}  softmax {e_sm:.3f}  preds {e_pr:.3f}')
    assert e_vol <= 1 and e_sm <= 1 and e_pr <= 1, (e_vol, e_sm, e_pr)
