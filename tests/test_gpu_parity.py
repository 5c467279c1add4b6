"""GPU parity tests (run with ``-m gpu`` on an H100): the CUDA path, called through
the C-ABI library, against the oracle / the reference-generated golden fixtures /
plain fp32 PyTorch ops, plus size-independent properties at the BASELINE.json shape.

Tolerance: BASELINE.json's north_star states 1e-3 relative (fp32).  We use the
normalised max-norm error  max|a-b| / max|b| <= 1e-3  for end-to-end outputs, and
much tighter bounds for single ops.
"""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import synthetic as syn
from oracle import dfm_oracle as O
from tests.util import (GOLDEN, KITTI_CASES, assert_close, load_kitti_case,
                        make_neck_mt_case, rel_err)

pytestmark = pytest.mark.gpu

TOL = 1e-3  # north_star tolerance


@pytest.fixture(scope='module', autouse=True)
def _fp32_reference():
    assert torch.cuda.is_available(), 'GPU tests need an H100'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _backbone(params, cfg, impl):
    m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg, conv_impl=impl).cuda().eval()
    m.load_state_dict(params, strict=True)
    m.downsampled_depth = O.downsampled_depth(cfg)
    return m


def test_library_loads_and_sees_h100():
    L = capi.lib()
    import ctypes
    sm, maj, mnr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    l2 = ctypes.c_longlong()
    capi.check(L.dfm_device_info(ctypes.byref(sm), ctypes.byref(maj),
                                 ctypes.byref(mnr), ctypes.byref(l2)), 'info')
    assert maj.value == 9 and sm.value >= 100


@pytest.mark.parametrize('name', sorted(KITTI_CASES))
def test_cost_volume_matches_reference(name):
    cur, prev, metas, params, cfg, gold = load_kitti_case(name)
    spec = KITTI_CASES[name]
    vol = modules.build_dfm_cost(
        cur.cuda(), prev.cuda(), O.downsampled_depth(cfg), 1, 4,
        torch.as_tensor(np.array([metas[0]['ori_cam2img']])),
        metas[0]['cur2prevs'], metas[0]['ori_shape'][:2], spec[4],
        metas[0]['crop_offset'], img_scale_factor=spec[6])
    ref = torch.from_numpy(gold['volume'])
    assert vol.shape == ref.shape
    assert rel_err(vol, ref) < TOL
    # cur half is the exact stride-4 subsample of the cur feature
    assert torch.equal(vol[0, :32, 3].cpu(), cur[0, :, ::4, ::4])


CONV_CASES = [
    # cin, cout, (D,H,W), stride, pad, transposed
    (32, 32, (6, 9, 21), (1, 1, 1), (1, 1, 1), False),
    (64, 32, (4, 8, 16), (1, 1, 1), (1, 1, 1), False),
    (32, 64, (8, 12, 20), (2, 2, 2), (1, 1, 1), False),
    (64, 64, (4, 6, 10), (1, 1, 1), (1, 1, 1), False),
    (64, 64, (8, 8, 12), (2, 2, 2), (1, 1, 1), False),
    (64, 64, (3, 4, 5), (2, 2, 2), (1, 1, 1), True),
    (64, 32, (4, 5, 7), (2, 2, 2), (1, 1, 1), True),
    (64, 128, (5, 4, 12), (1, 1, 2), (1, 1, 1), False),
    (128, 128, (4, 3, 6), (1, 1, 1), (1, 1, 1), False),
    (128, 256, (4, 3, 6), (1, 1, 2), (1, 1, 1), False),
    (256, 256, (4, 3, 3), (1, 1, 1), (1, 1, 0), False),
    # the BEV-neck kernel (conv_tc_neck.cuh) on grids larger than one 16 x 8 tile, one case
    # per z mode: stride (1,1,1) pad 1, stride (1,1,2), pad (1,1,0)
    (64, 64, (37, 21, 12), (1, 1, 1), (1, 1, 1), False),
    (128, 128, (35, 19, 6), (1, 1, 1), (1, 1, 1), False),
    (64, 128, (33, 26, 12), (1, 1, 2), (1, 1, 1), False),
    (128, 256, (18, 17, 6), (1, 1, 2), (1, 1, 1), False),
    (256, 256, (20, 23, 3), (1, 1, 1), (1, 1, 0), False),
]


@pytest.mark.parametrize('impl', ['simt', 'auto'])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv3d_op_vs_torch(case, impl):
    cin, cout, dims, stride, pad, tr = case
    g = torch.Generator().manual_seed(cin * 1000 + cout + dims[0])
    x = torch.randn((1, cin) + dims, generator=g).cuda()
    if tr:
        w = torch.randn((cin, cout, 3, 3, 3), generator=g) * 0.05
        ref = F.conv_transpose3d(x, w.cuda(), None, 2, 1, 1)
    else:
        w = torch.randn((cout, cin, 3, 3, 3), generator=g) * 0.05
        ref = F.conv3d(x, w.cuda(), None, stride, pad)
    y = modules.conv3d(x, w, stride, pad, tr, impl=impl)
    assert y.shape == ref.shape
    # simt: fp32 FMA chains; auto: bf16x2 split operands on the tensor cores
    assert rel_err(y, ref) < (2e-5 if impl == 'simt' else 1e-4)


@pytest.mark.parametrize('case', [c for c in CONV_CASES
                                  if not c[5] and c[0] >= 64 and c[2][2] <= 16 and c[3][:2] == (1, 1)])
def test_neck_conv_kernel_vs_torch(case):
    """The K-outer wgmma kernel of the BEV necks (conv_tc_neck.cuh), forced, on every shape
    it serves -- including the multi-tile grids -- against F.conv3d with TF32 off."""
    cin, cout, dims, stride, pad, _ = case
    g = torch.Generator().manual_seed(cin * 1000 + cout + dims[0])
    x = torch.randn((1, cin) + dims, generator=g).cuda()
    w = torch.randn((cout, cin, 3, 3, 3), generator=g) * 0.05
    ref = F.conv3d(x, w.cuda(), None, stride, pad)
    _, tc0 = capi.launch_counters()
    y = modules.conv3d(x, w, stride, pad, False, impl='tc_neck')
    _, tc1 = capi.launch_counters()
    assert tc1 == tc0 + 1
    assert y.shape == ref.shape
    e = rel_err(y, ref)
    print('neck kernel', case, e)
    assert e < 1e-4


def _windowed_k_outer_case(cin, cout, dims, zc, tpi, cg16, monkeypatch):
    if zc:
        monkeypatch.setenv('DFM_NECK_ZC', str(zc))
        monkeypatch.setenv('DFM_NECK_ZTPI', str(tpi))
    if cg16:    # weight images of 16 input x 64 output channels (N = 128 MMAs) where they fit
        if cout % 64:
            pytest.skip('the 16 / 64 group shape needs a multiple of 64 output channels')
        monkeypatch.setenv('DFM_NTK_CG16', '1')
    g = torch.Generator().manual_seed(cin * 1000 + cout + dims[0] + zc)
    x = torch.randn((1, cin) + dims, generator=g).cuda()
    w = torch.randn((cout, cin, 3, 3, 3), generator=g) * 0.05
    ref = F.conv3d(x, w.cuda(), None, 1, 1)
    _, tc0 = capi.launch_counters()
    y = modules.conv3d(x, w, (1, 1, 1), (1, 1, 1), False, impl='tc_neck_dhw')
    _, tc1 = capi.launch_counters()
    assert tc1 == tc0 + 1
    assert y.shape == ref.shape
    e = rel_err(y, ref)
    print('windowed K-outer kernel', cin, cout, dims, zc, tpi, cg16, e)
    assert e < 1e-4
    assert_close(y, ref, 'windowed conv')


@pytest.mark.parametrize('cg16', [False, True])
@pytest.mark.parametrize('zc,tpi', [(0, 0), (4, 1), (4, 4), (7, 2), (16, 1)])
@pytest.mark.parametrize('cin,cout,dims', [(64, 64, (19, 37, 21)), (64, 32, (9, 16, 8)),
                                           (128, 64, (33, 20, 30))])
def test_windowed_k_outer_conv_vs_torch(cin, cout, dims, zc, tpi, cg16, monkeypatch):
    """conv_tc_neck.cuh in plane-sweep-volume orientation ([D][H][W], D cut into windows whose
    halo planes are real data), forced, against F.conv3d with TF32 off, on ragged tile grids.
    Window lengths / tiles per item beyond the accumulator capacity (NK_ACC_COLS columns:
    4 planes x 32 channels or 2 x 64) are capped by the launcher; these requests check that the
    capped launch is still exact.  Shapes inside the capacity:
    test_windowed_k_outer_conv_window_shapes."""
    _windowed_k_outer_case(cin, cout, dims, zc, tpi, cg16, monkeypatch)


# (group shape, window length, tiles per item) within the accumulator capacity NK_ACC_COLS:
# 4 planes x 32 channels, or 2 planes x 64 channels; (0, 0): the plan of neck_dhw_plan
@pytest.mark.parametrize('cg16,zc,tpi', [(False, 0, 0), (False, 1, 4), (False, 2, 2),
                                         (False, 3, 1), (False, 4, 1),
                                         (True, 0, 0), (True, 1, 2), (True, 2, 1)])
@pytest.mark.parametrize('cin,cout,dims', [(64, 64, (19, 37, 21)), (64, 32, (9, 16, 8)),
                                           (128, 64, (32, 20, 30))])
def test_windowed_k_outer_conv_window_shapes(cin, cout, dims, zc, tpi, cg16, monkeypatch):
    """The windowed K-outer conv with every window length and tiles-per-item that fits the
    accumulators: window lengths that do (D = 9 for 1 and 3, D = 32 for 1, 2, 4) and do not
    (D = 19) divide D, several tiles per weight image (9 and 8 tiles in the first and last
    volume)."""
    _windowed_k_outer_case(cin, cout, dims, zc, tpi, cg16, monkeypatch)


@pytest.mark.parametrize('impl', ['simt', 'auto'])
@pytest.mark.parametrize('name', sorted(KITTI_CASES))
def test_backbone_matches_reference_fixture(name, impl):
    cur, prev, metas, params, cfg, gold = load_kitti_case(name)
    m = _backbone(params, cfg, impl)
    with torch.no_grad():
        cost, stereo, mono = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    capi.sync_check()
    for got, key in ((cost, 'cost'), (stereo, 'stereo'), (mono, 'mono')):
        ref = torch.from_numpy(gold[key])
        assert got.shape == ref.shape
        e = rel_err(got, ref)
        print(name, impl, key, 'rel err', e, 'worst element / tol', assert_close(got, ref, key))
        assert e < TOL, (key, e)
    launches, tc = capi.launch_counters()
    assert launches > 0


@pytest.mark.parametrize('name', sorted(KITTI_CASES))
def test_depth_head_matches_reference_fixture(name):
    cur, prev, metas, params, cfg, gold = load_kitti_case(name)
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2,
                       max_depth=59.6), with_convs=False, num_views=1,
        depth_loss=dict(type='balanced_focal', loss_weight=1.0, fg_weight=5,
                        bg_weight=1, alpha=1, gamma=2))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = 4
    cost = torch.from_numpy(gold['cost']).cuda()
    vol, sm, preds = head(cost)
    rvol, rsm, rpreds = O.depth_head_forward(torch.from_numpy(gold['cost']),
                                             O.depth_samples(cfg))
    assert rel_err(vol, rvol) < 1e-5
    assert float((sm.cpu() - rsm).abs().max()) < 1e-6
    assert rel_err(preds, torch.from_numpy(gold['depth_preds'])) < 1e-5
    assert rel_err(preds, rpreds) < 1e-5
    _, _, p2 = head(cost, return_volumes=False)
    assert torch.equal(p2, preds)


@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_backbone_midsize_vs_oracle(impl):
    # config[0]-like case the CPU oracle finishes in seconds: D=16 planes
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(5, h, w, d)
    cfg = syn.depth_cfg_for(d)
    with torch.no_grad():
        rcost, rst, rmo = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
    m = _backbone(params, cfg, impl)
    with torch.no_grad():
        cost, st, mo = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    capi.sync_check()
    for got, ref, key in ((cost, rcost, 'cost'), (st, rst, 'stereo'), (mo, rmo, 'mono')):
        e = rel_err(got, ref)
        print(impl, key, e)
        assert e < TOL, (key, e)


def test_shipped_kitti_config_shape_vs_oracle():
    # configs/dfm/dfm_r34_1x8_kitti-3d-3class.py as shipped: 320x1280 crops, num_bins 288 ->
    # D = 72 planes.  One whole frame through the CPU oracle (~10-20 s on the box's cores)
    # against the tensor-core path with all shortcuts (z-class first layer, shortened mono
    # tower) active.
    h, w, d = 320, 1280, 72
    cur, prev, metas, params = syn.make_kitti_pair(21, h, w, d, ori_shape=(375, 1242, 3),
                                                   crop_offset=(0, 55))
    cfg = syn.depth_cfg_for(d)
    torch.set_num_threads(max(1, (os.cpu_count() or 8)))
    with torch.no_grad():
        ref = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
    m = _backbone(params, cfg, 'auto')
    with torch.no_grad():
        out = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    capi.sync_check()
    for got, r, key in zip(out, ref, ('cost', 'stereo', 'mono')):
        e = rel_err(got, r)
        print('shipped-shape', key, e, 'worst element / tol', assert_close(got, r, key))
        assert e < TOL, (key, e)


def test_simt_and_tensor_core_paths_agree():
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(6, h, w, d)
    cfg = syn.depth_cfg_for(d)
    outs = {}
    for impl in ('simt', 'auto'):
        m = _backbone(params, cfg, impl)
        with torch.no_grad():
            outs[impl] = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    for a, b in zip(outs['simt'], outs['auto']):
        assert rel_err(a, b) < 2e-4


def test_z_shortened_mono_tower_equals_full_computation():
    # SURVEY.md section 7 shortcut: the mono tower is z-invariant away from the two z ends,
    # so it is computed on 16 + 8 + 16 planes and expanded.  Must equal the full computation.
    h, w, d = 64, 128, 64
    cur, prev, metas, params = syn.make_kitti_pair(8, h, w, d)
    cfg = syn.depth_cfg_for(d)
    outs = {}
    for key, env in (('short', None), ('full', '1')):
        if env is None:
            os.environ.pop('DFM_NO_ZSHORTEN', None)
        else:
            os.environ['DFM_NO_ZSHORTEN'] = env
        try:
            m = _backbone(params, cfg, 'auto')
            with torch.no_grad():
                outs[key] = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
            capi.sync_check()
        finally:
            os.environ.pop('DFM_NO_ZSHORTEN', None)
    for a, b, name in zip(outs['short'], outs['full'], ('cost', 'stereo', 'mono')):
        e = rel_err(a, b)
        print(name, e)
        assert e < 2e-5, (name, e)
    # and both agree with the fp32 SIMT path (no shortcut of any kind)
    m = _backbone(params, cfg, 'simt')
    with torch.no_grad():
        ref = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    for a, b in zip(outs['short'], ref):
        assert rel_err(a, b) < 2e-4


def test_error_behaviour():
    cfg = syn.depth_cfg_for(8)
    m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg).cuda().eval()
    cur = torch.zeros(1, 32, 32, 64)
    meta = [syn.make_img_meta(32, 64)]
    with pytest.raises(RuntimeError):  # CPU tensors: there is no CPU path
        m(cur, cur, meta)
    with pytest.raises(AssertionError):  # the reference supports B=1 only
        m(torch.zeros(2, 32, 32, 64).cuda(), torch.zeros(2, 32, 32, 64).cuda(), meta)
    with pytest.raises(RuntimeError):  # Ho = 36/4 = 9 is not a multiple of 4
        m(torch.zeros(1, 32, 36, 64).cuda(), torch.zeros(1, 32, 36, 64).cuda(),
          [syn.make_img_meta(36, 64)])


# ---------------------------------------------------------------------------
# BASELINE.json shape: 370x1224 padded to 384x1248, D=112 -- size-independent
# properties (the CPU oracle would need ~15 s per frame here)
# ---------------------------------------------------------------------------
@pytest.fixture(scope='module')
def full_size():
    h, w, d = 384, 1248, 112
    cur, prev, metas, params = syn.make_kitti_pair(3, h, w, d,
                                                   ori_shape=(370, 1224, 3))
    cfg = syn.depth_cfg_for(d)
    m = _backbone(params, cfg, 'auto')
    with torch.no_grad():
        out = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    capi.sync_check()
    return dict(m=m, cur=cur, prev=prev, metas=metas, cfg=cfg, out=out, d=d, h=h, w=w,
                params=params)


def test_full_size_matches_oracle(full_size):
    """THE benchmarked configuration (BASELINE.json configs[1]: 370x1224 padded to 384x1248,
    D=112): DfMBackbone + DepthHead on the tensor-core path with every shortcut on (z-class
    first layer, shortened mono tower, K-slice stride-2 convs) against one whole frame of the
    CPU oracle (dfm_backbone.py:143-214, depth_head.py:190-212), all three backbone outputs
    and depth_preds, max-norm and element-wise."""
    torch.set_num_threads(max(1, (os.cpu_count() or 8)))
    cfg = full_size['cfg']
    with torch.no_grad():
        ref = O.dfm_backbone_forward(full_size['params'], full_size['cur'], full_size['prev'],
                                     full_size['metas'], cfg)
        rpred = O.depth_head_forward(ref[0], O.depth_samples(cfg))[2]
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2, max_depth=59.6),
        with_convs=False, num_views=1, depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = 4
    pred = head(full_size['out'][0], return_volumes=False)[2]
    for got, r, key in zip(tuple(full_size['out']) + (pred,), tuple(ref) + (rpred,),
                           ('cost', 'stereo', 'mono', 'depth_preds')):
        e = rel_err(got, r)
        print('D=112 384x1248', key, 'rel err', e, 'worst element / tol',
              assert_close(got, r, key))
        assert e < TOL, (key, e)


def test_white_noise_features_vs_oracle():
    """Non-smooth inputs: relu(white noise) features have O(1) differences between
    neighbouring pixels, so any sampling-coordinate difference between the closed-form warp /
    exact-lattice cur half and the reference's fp32 pixel -> 3-D -> pixel round trip shows
    up undamped (SURVEY.md section 7).  Crop + scale so the lattice is off the pixel grid of
    the original image; checked at the outputs, as north_star states the tolerance."""
    h, w, d = 128, 256, 16
    rng = np.random.RandomState(17)
    cur = torch.from_numpy(rng.standard_normal((1, 32, h, w)).astype(np.float32)).relu()
    prev = torch.from_numpy(rng.standard_normal((1, 32, h, w)).astype(np.float32)).relu()
    _, _, metas, params = syn.make_kitti_pair(17, h, w, d, crop_offset=(400, 100), scale=1.0,
                                              ori_shape=(375, 1242, 3))
    cfg = syn.depth_cfg_for(d)
    with torch.no_grad():
        ref = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
    for impl in ('auto', 'simt'):
        m = _backbone(params, cfg, impl)
        with torch.no_grad():
            out = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        capi.sync_check()
        for got, r, key in zip(out, ref, ('cost', 'stereo', 'mono')):
            e = rel_err(got, r)
            print('white-noise', impl, key, e)
            assert e < TOL, (key, e)


def test_full_size_outputs_finite_and_shaped(full_size):
    cost, st, mo = full_size['out']
    d = full_size['d']
    assert cost.shape == (1, 1, d, 96, 312)
    assert st.shape == (1, 32, d, 96, 312) and mo.shape == st.shape
    for t in (cost, st, mo):
        assert bool(torch.isfinite(t).all())
    assert float(st.std()) > 0.1


def test_full_size_mono_tower_ignores_prev_frame(full_size):
    # the mono tower sees cost_raw[:, :32] only (dfm_backbone.py:189)
    m = full_size['m']
    prev2 = torch.roll(full_size['prev'], 7, dims=-1).cuda()
    with torch.no_grad():
        cost2, st2, mo2 = m(full_size['cur'].cuda(), prev2,
                            copy.deepcopy(full_size['metas']))
    assert torch.equal(mo2, full_size['out'][2])
    assert not torch.equal(st2, full_size['out'][1])


def test_full_size_identity_pose_volume_is_subsample():
    # cur2prev = I  =>  the warp is the identity: both halves of the volume are the
    # stride-4 subsample of their feature map on every plane
    h, w, d = 384, 1248, 112
    rng = np.random.RandomState(9)
    cur = syn.smooth_field(rng, 32, h, w).cuda()
    prev = syn.smooth_field(rng, 32, h, w).cuda()
    meta = syn.make_img_meta(h, w, ori_shape=(370, 1224, 3))
    meta['cur2prevs'] = torch.eye(4)[None]
    cfg = syn.depth_cfg_for(d)
    vol = modules.build_dfm_cost(cur, prev, O.downsampled_depth(cfg), 1, 4,
                                 torch.as_tensor(np.array([meta['ori_cam2img']])),
                                 meta['cur2prevs'], (370, 1224))
    assert vol.shape == (1, 64, d, 96, 312)
    sub_c = cur[0, :, ::4, ::4]
    sub_p = prev[0, :, ::4, ::4]
    for z in (0, 55, 111):
        assert torch.equal(vol[0, :32, z], sub_c)
        assert float((vol[0, 32:, z] - sub_p).abs().max()) < 2e-3


def test_full_size_depth_head_properties(full_size):
    cfg = full_size['cfg']
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2,
                       max_depth=59.6), with_convs=False, num_views=1,
        depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = 4
    vol, sm, preds = head(full_size['out'][0])
    assert sm.shape == (1, 1, 448, 384, 1248)
    s = sm.sum(2)
    assert float((s - 1).abs().max()) < 1e-4
    assert float(preds.min()) > 2.0 and float(preds.max()) < 59.6
    # trilinear with align_corners reproduces the low-res logits at the corners
    c = full_size['out'][0]
    assert torch.allclose(vol[0, 0, 0, 0, 0], c[0, 0, 0, 0, 0])
    assert torch.allclose(vol[0, 0, -1, -1, -1], c[0, 0, -1, -1, -1])
    e = (sm * head.depth_samples.cuda()[None, None, :, None, None]).sum(2)
    assert rel_err(preds, e) < 1e-5


# ---------------------------------------------------------------------------
# Waymo path: lifting + necks
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['neck_dfm', 'neck_imvoxel'])
@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_neck_matches_reference_fixture(name, impl):
    gold = np.load(os.path.join(GOLDEN, name + '.npz'))
    rng = np.random.RandomState(21)
    dfm = modules.DfMNeck(64, 256, num_frames=2, conv_impl=impl)
    imv = modules.OutdoorImVoxelNeck(64, 256, conv_impl=impl)
    sd_dfm = syn.make_neck_params(rng, dfm.state_dict())
    rng.standard_normal((1, 128, 6, 5, 12))
    sd_imv = syn.make_neck_params(rng, imv.state_dict())
    mod, sd = (dfm, sd_dfm) if name == 'neck_dfm' else (imv, sd_imv)
    mod.load_state_dict(sd, strict=True)
    mod = mod.cuda().eval()
    y = mod(torch.from_numpy(gold['x']).cuda())[0]
    ref = torch.from_numpy(gold['y'])
    assert y.shape == ref.shape
    e = rel_err(y, ref)
    print(name, impl, e)
    assert e < TOL


@pytest.mark.parametrize('name', ['neck_dfm_mt', 'neck_imvoxel_mt'])
@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_neck_multitile_matches_reference_fixture(name, impl):
    """The necks on 37 x 21 x 12 voxels (3 x 3 tiles of the K-outer tensor-core kernel, ragged
    right/bottom tiles) against the verbatim reference output: tile seams, the per-group weight
    reload across tiles and the stride-(1,1,2) / pad-(1,1,0) layers at Nz = 12 -> 6 -> 3 -> 1."""
    gold = np.load(os.path.join(GOLDEN, name + '.npz'))
    rng, x = make_neck_mt_case(name)
    mod = (modules.DfMNeck(64, 256, num_frames=2, conv_impl=impl) if name == 'neck_dfm_mt'
           else modules.OutdoorImVoxelNeck(64, 256, conv_impl=impl))
    mod.load_state_dict(syn.make_neck_params(rng, mod.state_dict()), strict=True)
    mod = mod.cuda().eval()
    y = mod(x.cuda())[0]
    capi.sync_check()
    ref = torch.from_numpy(gold['y'])
    assert y.shape == ref.shape
    e = rel_err(y, ref)
    print(name, impl, e, 'worst element / tol', assert_close(y, ref, name))
    assert e < TOL


def _lift_case(concat, flip):
    rng = np.random.RandomState(31)
    t, nv, c, hf, wf = 2, 3, 64, 20, 32
    in_h, in_w = 80, 128
    feats = torch.from_numpy(rng.standard_normal((t * nv, c, hf, wf)).astype(np.float32))
    n_voxels = [12, 10, 4]
    vrange = [2.0, -10.0, -2.0, 26.0, 10.0, 2.0]
    mats = []
    for f in range(t):
        for v in range(nv):
            yaw = (v - 1) * 0.6
            # camera looks along +x (lidar frame), yawed; x_cam = -y_l, y_cam = -z_l, z_cam = x_l
            r = np.array([[np.cos(yaw), np.sin(yaw), 0], [-np.sin(yaw), np.cos(yaw), 0],
                          [0, 0, 1]])
            l2c = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64) @ r
            ext = np.eye(4)
            ext[:3, :3] = l2c
            ext[:3, 3] = l2c @ np.array([-0.5 * f, 0.1 * v, 0.3])
            k = np.array([[60., 0, 64, 0], [0, 60., 40, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
            mats.append(k @ ext)
    meta = dict(ori_lidar2img=np.array(mats), input_shape=(in_h, in_w), _feat_hw=(hf, wf),
                img_shape=[(in_h - 2, in_w - 3, 3)] * (t * nv),
                scale_factor=np.array([0.98, 1.01, 0.98, 1.01], dtype=np.float32),
                img_crop_offset=[1.5, 0.5], flip=flip)
    return feats, meta, n_voxels, vrange, t, nv


@pytest.mark.parametrize('concat', [False, True])
@pytest.mark.parametrize('flip', [False, True])
def test_multiview_lift_vs_oracle(concat, flip):
    feats, meta, n_voxels, vrange, t, nv = _lift_case(concat, flip)
    agg = 'concat' if concat else 'mean'
    got = modules.multiview_lift(feats.cuda(), meta, n_voxels, vrange, nv, t, agg)
    xs, ys, zs = modules.aligned_voxel_centers(n_voxels, vrange)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
    l2i = [torch.tensor(m, dtype=torch.float32) for m in meta['ori_lidar2img']]
    ref = O.multiview_lift(feats, pts, n_voxels, l2i, nv, t,
                           pts.new_tensor(meta['scale_factor'][:2]),
                           pts.new_tensor(meta['img_crop_offset']), flip,
                           meta['input_shape'], meta['img_shape'], agg)
    assert got.shape == ref.shape
    # index work: the kernel reproduces the reference's fp32 rounding sequence
    # (lift_project in simt_kernels.cuh), so every voxel picks the same tap
    bad = _lift_mismatches(got.cpu(), ref, pts, meta, t * nv)
    assert bad == 0, bad
    assert float(ref.abs().sum()) > 0


def _lift_mismatches(got, ref, pts, meta, nsamp, tol_px=2e-3):
    """Number of voxels whose lifted features differ from the oracle's; every one of them
    must be explained by a view whose (fp64) projection sits within tol_px of a nearest-tap
    rounding tie or of a validity boundary -- anything else is a bug, not rounding."""
    diff = (got - ref).abs().amax(0).reshape(-1)            # [Nx*Ny*Nz] in output order
    scale = float(ref.abs().max())
    nx, ny, nz = ref.shape[1:]
    bad = torch.nonzero(diff > 1e-5 * scale).reshape(-1)
    if bad.numel() == 0:
        return 0
    # output order is [Nx][Ny][Nz]; pts are z-major, then y, then x fastest
    ix, iy, iz = bad // (ny * nz), (bad // nz) % ny, bad % nz
    p = pts[(iz * ny + iy) * nx + ix].double()
    in_h, in_w = meta['input_shape'][:2]
    hf, wf = 0, 0
    explained = torch.zeros(bad.numel(), dtype=torch.bool)
    sf = np.asarray(meta['scale_factor'], dtype=np.float64)
    crop = np.asarray(meta.get('img_crop_offset', (0, 0)), dtype=np.float64)
    for s in range(nsamp):
        m = torch.tensor(np.asarray(meta['ori_lidar2img'][s], dtype=np.float32),
                         dtype=torch.float64)
        q = torch.cat([p, torch.ones(len(p), 1, dtype=torch.float64)], 1) @ m.T
        cx = q[:, 0] / q[:, 2] * sf[0] - crop[0]
        cy = q[:, 1] / q[:, 2] * sf[1] - crop[1]
        if meta.get('flip', False):
            cx = meta['img_shape'][s][1] - cx
        hf, wf = meta['_feat_hw']
        fx, fy = cx / in_w * (wf - 1), cy / in_h * (hf - 1)
        tie = ((fx - fx.floor() - 0.5).abs() < tol_px) | ((fy - fy.floor() - 0.5).abs() < tol_px)
        edge = (cx.abs() < tol_px) | ((cx - in_w).abs() < tol_px) | (cy.abs() < tol_px) | \
            ((cy - in_h).abs() < tol_px) | (q[:, 2].abs() < 1e-4)
        explained |= tie | edge
    assert bool(explained.all()), \
        f'{int((~explained).sum())} of {bad.numel()} mismatching voxels are not rounding ties'
    return int(bad.numel())


@pytest.mark.parametrize('t,agg', [(1, 'mean'), (2, 'concat'), (2, 'mean')])
def test_multiview_lift_full_size_exact(t, agg):
    """Waymo size (configs/dfm/multiview-dfm_*: 220 x 300 x 12 voxels, T x 5 views of
    [64, 208, 312] features): the lifted volume equals the oracle's voxel for voxel."""
    nv = 5
    feats, meta = syn.make_waymo_sample(40 + t, t, nv)
    meta['_feat_hw'] = tuple(feats.shape[-2:])
    n_voxels, vrange = syn.WAYMO_N_VOXELS, syn.WAYMO_RANGE
    got = modules.multiview_lift(feats.cuda(), meta, n_voxels, vrange, nv, t, agg)
    xs, ys, zs = modules.aligned_voxel_centers(n_voxels, vrange)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
    l2i = [torch.tensor(m, dtype=torch.float32) for m in meta['ori_lidar2img']]
    torch.set_num_threads(max(1, (os.cpu_count() or 8)))
    ref = O.multiview_lift(feats, pts, n_voxels, l2i, nv, t,
                           pts.new_tensor(meta['scale_factor'][:2]),
                           pts.new_tensor(meta['img_crop_offset']), False,
                           meta['input_shape'], meta['img_shape'], agg)
    assert got.shape == ref.shape == (64 * (t if agg == 'concat' else 1), 220, 300, 12)
    # channels-last memory (what the necks read); the reference-layout entry point gives the
    # same bits
    assert got.permute(1, 2, 3, 0).is_contiguous()
    got_ncdhw = modules.multiview_lift(feats.cuda(), meta, n_voxels, vrange, nv, t, agg,
                                       channels_last=False)
    assert got_ncdhw.is_contiguous() and torch.equal(got_ncdhw, got)
    del got_ncdhw
    bad = _lift_mismatches(got.cpu(), ref, pts, meta, t * nv)
    nonzero = float((ref.abs().amax(0) > 0).float().mean())
    print(f'lift T={t} {agg}: {bad} mismatching voxels of {pts.shape[0]}, '
          f'{100 * nonzero:.1f} % of voxels see a camera')
    assert bad == 0
    assert nonzero > 0.2


# ---------------------------------------------------------------------------
# FrustumToVoxel (SURVEY.md section 8(f) row 1)
# ---------------------------------------------------------------------------
def _frustum_module(c, impl='auto', **kw):
    m = modules.FrustumToVoxel(conv_impl=impl, **kw)
    m.load_state_dict(c['params'], strict=True)
    m = m.cuda().eval()
    m.coordinates_3d = c['coordinates_3d']
    m.depth_cfg = c['depth_cfg']
    return m


@pytest.mark.parametrize('impl', ['simt', 'auto'])
@pytest.mark.parametrize('fused', [False, True])
def test_frustum_matches_reference_fixture(impl, fused):
    """CUDA FrustumToVoxel vs the verbatim reference run (tests/golden/frustum.npz): with the
    reference's materialised softmax volume, and with the volume rebuilt from the logits."""
    from tests.util import load_frustum_case
    c, gold = load_frustum_case()
    m = _frustum_module(c, impl)
    dist = (modules.CostLogits(c['cost'].cuda()) if fused
            else torch.from_numpy(gold['softmax']).cuda())
    out = m(c['stereo'].cuda(), dist, c['metas'], c['sem'].cuda())
    ref = torch.from_numpy(gold['out'])
    assert out.shape == ref.shape
    e = rel_err(out, ref)
    print('frustum fixture', impl, fused, e)
    assert e < TOL


@pytest.mark.parametrize('variant', ['default', 'stereo_atten', 'no_img', 'two_convs'])
def test_frustum_variants_vs_oracle(variant):
    """Constructor switches (feature_transformation.py:17-22) and a voxel grid that leaves
    the depth range and the image on all sides, against the oracle."""
    kw = dict(default={}, stereo_atten=dict(stereo_atten_feat=True, sem_atten_feat=False),
              no_img=dict(cat_img_feature=False, stereo_atten_feat=True),
              two_convs=dict(num_3dconvs=2))[variant]
    c = syn.make_frustum_case(41, 64, 160, 12, (40, 36, 12),
                              num_3dconvs=kw.get('num_3dconvs', 1),
                              cat_img_feature=kw.get('cat_img_feature', True))
    # grid from 0.5 m (closer than depth_min) to 70 m (beyond depth_max)
    c['coordinates_3d'] = syn.frustum_coordinates([0.5, -30.4, -3, 70.0, 30.4, 1],
                                                  (40, 36, 12))
    cfg = c['depth_cfg']
    _, sm, _ = O.depth_head_forward(c['cost'], O.depth_samples(cfg), 4)
    ref = O.frustum_to_voxel_forward(
        c['params'], c['stereo'], sm, c['metas'], c['sem'], c['coordinates_3d'], cfg,
        sem_atten_feat=kw.get('sem_atten_feat', True),
        stereo_atten_feat=kw.get('stereo_atten_feat', False),
        cat_img_feature=kw.get('cat_img_feature', True),
        num_3dconvs=kw.get('num_3dconvs', 1))
    m = _frustum_module(c, **kw)
    sem = c['sem'].cuda() if kw.get('cat_img_feature', True) else None
    a = m(c['stereo'].cuda(), sm.cuda(), c['metas'], sem)
    b = m(c['stereo'].cuda(), modules.CostLogits(c['cost'].cuda()), c['metas'], sem)
    ea, eb = rel_err(a, ref), rel_err(b, ref)
    print('frustum', variant, ea, eb, float((ref != 0).float().mean()))
    assert ea < TOL and eb < TOL


def test_frustum_full_size_properties():
    """KITTI shape (D=112 planes, 96x312 lattice, 20x304x288 voxels): the fused path
    agrees with the materialised-softmax path, voxels that project outside the image carry
    only the conv's response to zeros, and the output is finite."""
    c = syn.make_frustum_case(51, 384, 1248, 112, (288, 304, 20))
    m = _frustum_module(c)
    stereo, cost, sem = c['stereo'].cuda(), c['cost'].cuda(), c['sem'].cuda()
    head = modules.DepthHead(depth_cfg=dict(mode='UD', num_bins=448, min_depth=2,
                                            max_depth=59.6), with_convs=False)
    head.depth_samples = O.depth_samples(c['depth_cfg'])
    _, sm, _ = head(cost)
    a = m(stereo, sm, c['metas'], sem)
    del sm
    b = m(stereo, modules.CostLogits(cost), c['metas'], sem)
    assert a.shape == (1, 32, 5, 304, 288)
    assert torch.isfinite(a).all()
    e = rel_err(b, a)
    print('frustum full size fused vs materialised', e)
    assert e < 1e-4
    # zero input region: y = +-30 m at x = 2.1 m projects far outside the image on every
    # height, and so do its 3x3x3 neighbours -> out = relu(gn(0)) there
    sc = m.voxel_convs[0][0].gn
    corner = a[0, :, :, 0, 0].cpu()
    # raw conv output 0 -> (0 - mean) * rstd * gamma + beta: identical on all pooled planes
    assert float((corner - corner[:, :1]).abs().max()) < 1e-5
    assert sc.weight.numel() == 32


def test_frustum_fused_depth_preds_and_backbone_twin():
    """backbone -> (DepthHead + FrustumToVoxel in one call): depth_preds of the fused pass
    equal the DepthHead's, and reading the backbone's channels-last twin of stereo_feat gives
    the same voxels as transposing the NCDHW tensor."""
    from tests.util import load_frustum_case
    cur, prev, metas, params, cfg, _ = load_kitti_case('kitti_plain')
    bb = _backbone(params, cfg, 'auto')
    cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    assert getattr(stereo, '_dfm_channels_last', None) is not None
    c, _ = load_frustum_case()
    m = _frustum_module(c)
    sem = c['sem'].cuda()
    samples = O.depth_samples(cfg)
    lg = modules.CostLogits(cost, depth_samples=samples)
    a = m(stereo, lg, c['metas'], sem)                      # twin path
    b = m(stereo.clone(), modules.CostLogits(cost), c['metas'], sem)  # transpose path
    assert torch.equal(a, b)
    _, sm, preds = O.depth_head_forward(cost.cpu(), samples, 4)
    assert rel_err(lg.depth_preds, preds) < 1e-5
    ref = O.frustum_to_voxel_forward(c['params'], stereo.cpu(), sm, c['metas'], c['sem'],
                                     c['coordinates_3d'], cfg)
    e = rel_err(a, ref)
    print('backbone -> frustum', e)
    assert e < TOL
    # a second backbone forward invalidates the twin: the module must fall back to the tensor
    bb(prev.cuda(), cur.cuda(), copy.deepcopy(metas))
    a2 = m(stereo, modules.CostLogits(cost), c['metas'], sem)
    assert torch.equal(a2, b)


def test_forward_host_and_prefetch_match_device_path():
    """dfm_backbone_forward_host (host buffers in/out) and the prefetched variant
    (dfm_backbone_prefetch_host for the next pair while the current one is processed) return
    what dfm_backbone_forward returns on device tensors."""
    import ctypes
    cur, prev, metas, params, cfg, _ = load_kitti_case('kitti_plain')
    m = _backbone(params, cfg, 'auto')
    cost, stereo, mono = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    torch.cuda.synchronize()
    L = capi.lib()
    g = modules.geometry_from_meta(metas[0])
    hc, hp = cur.contiguous().pin_memory(), prev.contiguous().pin_memory()
    hc2, hp2 = prev.contiguous().pin_memory(), cur.contiguous().pin_memory()
    outs = [torch.empty_like(t, device='cpu').pin_memory() for t in (cost, stereo, mono)]
    flags = capi.DFM_OUT_COST | capi.DFM_OUT_STEREO | capi.DFM_OUT_MONO
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(a, b):
        capi.check(L.dfm_backbone_forward_host(
            m._handle, ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr()),
            ctypes.byref(g), flags, *[ctypes.c_void_p(o.data_ptr()) for o in outs], stream),
            'dfm_backbone_forward_host')
        return [o.clone() for o in outs]

    def pf(a, b):
        capi.check(L.dfm_backbone_prefetch_host(
            m._handle, ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr())),
            'dfm_backbone_prefetch_host')

    plain = run(hc, hp)
    for got, ref in zip(plain, (cost, stereo, mono)):
        assert rel_err(got, ref) < 1e-5
    swapped = run(hc2, hp2)
    # prefetch both pairs, consume them in order, then once more with a stale third prefetch
    pf(hc, hp)
    pf(hc2, hp2)
    a = run(hc, hp)
    pf(hc, hp)
    b = run(hc2, hp2)
    c = run(hc, hp)
    for got, ref in zip(a, plain):
        assert rel_err(got, ref) < 1e-5
    for got, ref in zip(b, swapped):
        assert rel_err(got, ref) < 1e-5
    for got, ref in zip(c, plain):
        assert rel_err(got, ref) < 1e-5


def test_pipeline_forward_host_matches_module_path():
    """dfm_pipeline_forward_host (host buffers in/out: DfMBackbone -> DepthHead reduction ->
    FrustumToVoxel in one call, detectors/dfm.py:296,420,423-425) returns what the three mirror
    modules return on device tensors, with and without a prefetched pair, and matches the
    all-oracle pipeline."""
    from tests.util import load_frustum_case
    cur, prev, metas, params, cfg, _ = load_kitti_case('kitti_plain')
    c, _ = load_frustum_case()
    metas = copy.deepcopy(metas)
    metas[0]['cam2img'] = c['metas'][0]['cam2img']
    metas[0]['pad_shape'] = c['metas'][0]['pad_shape']
    bb = _backbone(params, cfg, 'auto')
    fr = _frustum_module(c)
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2, max_depth=59.6),
        with_convs=False, num_views=1, depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = 4
    sem = c['sem'].cuda()
    with torch.no_grad():
        cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        lg = modules.CostLogits(cost, depth_samples=head.depth_samples)
        vox_ref = fr(stereo, lg, metas, sem).cpu()
        pred_ref = lg.depth_preds.cpu()
    pipe = modules.HotPathPipeline(bb, head, fr)
    hc, hp = cur.contiguous().pin_memory(), prev.contiguous().pin_memory()
    hs = c['sem'].contiguous().pin_memory()
    h_cost = torch.empty((1, 1) + tuple(cost.shape[2:])).pin_memory()
    vox, pred = pipe(hc, hp, hs, metas, h_cost=h_cost)
    # (two runs of the backbone differ in the last bits: GroupNorm sums are fp64 atomics)
    assert rel_err(vox, vox_ref) < 1e-5 and rel_err(pred, pred_ref) < 1e-5
    assert rel_err(h_cost, cost) < 1e-5
    pipe.prefetch(hc, hp)
    vox2, pred2 = pipe(hc, hp, hs, metas)
    assert rel_err(vox2, vox_ref) < 1e-5 and rel_err(pred2, pred_ref) < 1e-5
    # sem features staged with the pair; a different sem tensor at call time is a miss for the
    # staged copy (the call's tensor wins)
    pipe.prefetch(hc, hp, hs)
    vox2, pred2 = pipe(hc, hp, hs, metas)
    assert rel_err(vox2, vox_ref) < 1e-5 and rel_err(pred2, pred_ref) < 1e-5
    hs_other = (hs * 0.5).contiguous().pin_memory()
    pipe.prefetch(hc, hp, hs_other)
    vox2, _ = pipe(hc, hp, hs, metas)
    assert rel_err(vox2, vox_ref) < 1e-5
    pipe.prefetch(hc, hp, hs_other)
    vox3, _ = pipe(hc, hp, hs_other, metas)
    assert rel_err(vox3, vox_ref) > 1e-3
    # asynchronous form: two frames in flight (cur/prev swapped for the second), results collected
    # in order; the first equals the synchronous result, the second differs from it
    vox_ref1 = pipe(hc, hp, hs, metas)[0].clone()   # (pinned outputs are overwritten by later calls)
    pipe.submit(hc, hp, hs, metas)
    pipe.submit(hp, hc, hs, metas)
    with pytest.raises(RuntimeError):          # at most two frames in flight
        pipe.submit(hc, hp, hs, metas)
    a_vox, a_pred = pipe.wait()
    a_vox, a_pred = a_vox.clone(), a_pred.clone()
    b_vox, _ = pipe.wait()
    assert rel_err(a_vox, vox_ref1) < 1e-5 and rel_err(a_pred, pred_ref) < 1e-5
    assert rel_err(b_vox, vox_ref1) > 1e-3
    vox, pred = pipe(hc, hp, hs, metas)
    # all-oracle pipeline
    with torch.no_grad():
        rc, rs, _ = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
        _, sm, rp = O.depth_head_forward(rc, O.depth_samples(cfg), 4)
        rv = O.frustum_to_voxel_forward(c['params'], rs, sm, metas, c['sem'],
                                        c['coordinates_3d'], cfg)
    e_v, e_p = rel_err(vox, rv), rel_err(pred, rp)
    print('pipeline vs oracle: voxel', e_v, 'depth_preds', e_p)
    assert e_v < TOL and e_p < TOL


@pytest.mark.parametrize('t,agg,neck', [(1, 'mean', 'imvoxel'), (2, 'concat', 'dfm')])
def test_multiview_feature_transformation_mixin_vs_oracle(t, agg, neck):
    """The MultiViewDfM.feature_transformation-compatible override (batch loop, img_metas keys,
    return tuple; detectors/multiview_dfm.py:119-268) against the oracle: lifting + neck_3d on a
    batch of two samples with different metas."""
    nv = 3
    n_voxels, vrange = [20, 18, 12], [0.0, -9.0, -2.0, 20.0, 9.0, 4.0]
    rng = np.random.RandomState(61)
    mod = (modules.DfMNeck(64, 256, num_frames=2) if neck == 'dfm'
           else modules.OutdoorImVoxelNeck(64, 256))
    sd = syn.make_neck_params(rng, mod.state_dict())
    mod.load_state_dict(sd, strict=True)
    mod = mod.cuda().eval()

    class Host(modules.MultiViewDfMFeatureTransformation):
        pass
    host = Host()
    host.n_voxels, host.voxel_range = n_voxels, vrange
    host.temporal_aggregate, host.valid_sample, host.neck_3d = agg, True, mod
    feats, metas = [], []
    for b in range(2):
        f, m = syn.make_waymo_sample(70 + b, t, nv, feat_hw=(40, 64), input_hw=(160, 256),
                                     flip=bool(b), scale=1.0 + 0.02 * b, crop=(1.0 * b, 2.0 * b))
        k = np.array([[120., 0, 128, 0], [0, 120., 80, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        full = syn.waymo_lidar2img(t, nv)
        kfull = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        m['ori_lidar2img'] = np.array([k @ np.linalg.inv(kfull) @ x for x in full])
        feats.append(f)
        metas.append(m)
    batch = torch.stack(feats).cuda()
    with torch.no_grad():
        out = host.feature_transformation(batch, metas, nv, t)
    assert isinstance(out, tuple) and len(out) == 1
    assert out[0].shape == (2, 256, n_voxels[1], n_voxels[0])
    xs, ys, zs = modules.aligned_voxel_centers(n_voxels, vrange)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
    for b in range(2):
        m = metas[b]
        l2i = [torch.tensor(x, dtype=torch.float32) for x in m['ori_lidar2img']]
        with torch.no_grad():
            vol = O.multiview_lift(feats[b], pts, n_voxels, l2i, nv, t,
                                   pts.new_tensor(m['scale_factor'][:2]),
                                   pts.new_tensor(m['img_crop_offset']), m['flip'],
                                   m['input_shape'], m['img_shape'], agg)[None]
            ref = (O.dfm_neck_forward(sd, vol, 64) if neck == 'dfm'
                   else O.imvoxel_neck_forward(sd, vol))[0]
        assert float(vol.abs().sum()) > 0
        e = rel_err(out[0][b], ref[0])
        print('feature_transformation', neck, b, e)
        assert e < TOL


# ---------------------------------------------------------------------------
# 2-D BEV stage: BEVHourglass + LIGAAnchor3DHead (SURVEY.md section 8(f) row 3) and the
# north_star's "3D box regressions match the reference"
# ---------------------------------------------------------------------------
def _bev_modules(c, impl='auto'):
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
                              rotations=[0, 1.57], reshape_out=False),
        bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'), conv_impl=impl)
    head.load_state_dict(c['head'], strict=True)
    return bev.cuda().eval(), head.cuda().eval()


@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_bev_stage_matches_reference_fixture(impl):
    """CUDA BEVHourglass + LIGAAnchor3DHead against the verbatim reference run
    (tests/golden/bev_stage.npz, 44 x 36 cells = 3 x 5 conv tiles with ragged edges)."""
    gold = np.load(os.path.join(GOLDEN, 'bev_stage.npz'))
    c = syn.make_bev_case(**syn.BEV_CASE)
    bev, head = _bev_modules(c, impl)
    v = c['volume'].cuda()
    x = v.view(1, -1, v.shape[3], v.shape[4])              # detectors/dfm.py:427-428
    _, tc0 = capi.launch_counters()
    prehg, feat = bev(x)                                   # :429
    cls, box, dirc = head([feat])                          # :432
    capi.sync_check()
    _, tc1 = capi.launch_counters()
    assert (tc1 - tc0 > 0) == (impl == 'auto')
    assert isinstance(cls, list) and len(cls) == 1
    for got, key in ((prehg, 'prehg'), (feat, 'bev'), (cls[0], 'cls_score'),
                     (box[0], 'bbox_pred'), (dirc[0], 'dir_cls_preds')):
        ref = torch.from_numpy(gold[key])
        e = rel_err(got, ref)
        print('bev stage', impl, key, e, 'worst element / tol', assert_close(got, ref, key))
        assert e < TOL, (key, e)


def test_bev_stage_full_size_vs_torch_gpu():
    """KITTI size (160 channels, 304 x 288 cells): the CUDA stage against the same reference
    ops run by PyTorch on the GPU with TF32 off."""
    c = syn.make_bev_case(seed=93, nz=5, ny=304, nx=288)
    bev, head = _bev_modules(c)
    v = c['volume'].cuda()
    x = v.view(1, 160, 304, 288)
    _, feat = bev(x)
    cls, box, dirc = head.forward_single(feat)
    capi.sync_check()
    pb = {k: t.cuda() for k, t in c['bev'].items()}
    ph = {k: t.cuda() for k, t in c['head'].items()}
    with torch.no_grad():
        _, rfeat = O.bev_hourglass_forward(pb, x)
        rcls, rbox, rdir = O.liga_anchor3d_head_forward(ph, rfeat)
    for got, ref, key in ((feat, rfeat, 'bev'), (cls, rcls, 'cls_score'),
                          (box, rbox, 'bbox_pred'), (dirc, rdir, 'dir_cls_preds')):
        e = rel_err(got, ref)
        print('bev stage 304x288', key, e, 'worst element / tol', assert_close(got, ref, key))
        assert e < TOL, (key, e)


def test_box_regression_parity_end_to_end():
    """north_star: "depth logits and 3D box regressions match the reference PyTorch path on
    identical inputs within 1e-3".  All-CUDA DfM.simple_test segment (detectors/dfm.py:416-432:
    DfMBackbone -> DepthHead/FrustumToVoxel -> height compression -> BEVHourglass ->
    LIGAAnchor3DHead) against the all-oracle pipeline on the same pair."""
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(23, h, w, d)
    cfg = syn.depth_cfg_for(d)
    fc = syn.make_frustum_case(24, h, w, d, (32, 28, 20))
    metas = copy.deepcopy(metas)
    metas[0]['cam2img'] = fc['metas'][0]['cam2img']
    bc = syn.make_bev_case(seed=25, nz=5, ny=28, nx=32)
    # ---- oracle ----
    with torch.no_grad():
        rcost, rstereo, _ = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
        _, sm, rpreds = O.depth_head_forward(rcost, O.depth_samples(cfg), 4)
        rvol = O.frustum_to_voxel_forward(fc['params'], rstereo, sm, metas, fc['sem'],
                                          fc['coordinates_3d'], cfg)
        rcls, rbox, rdir = O.dfm_bev_stage(bc['bev'], bc['head'], rvol)
    assert float((rvol != 0).float().mean()) > 0.2
    # ---- CUDA ----
    bb = _backbone(params, cfg, 'auto')
    fr = _frustum_module(fc)
    bev, head = _bev_modules(bc)
    with torch.no_grad():
        cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        lg = modules.CostLogits(cost, depth_samples=O.depth_samples(cfg))
        vol = fr(stereo, lg, metas, fc['sem'].cuda())
        _, nz, ny, nx = vol.shape[1:]
        _, feat = bev(vol.view(1, -1, ny, nx))
        cls, box, dirc = head([feat])
    capi.sync_check()
    for got, ref, key in ((cost, rcost, 'depth logits'), (lg.depth_preds, rpreds, 'depth_preds'),
                          (vol, rvol, 'voxel features'), (cls[0], rcls, 'cls_score'),
                          (box[0], rbox, 'bbox_pred'), (dirc[0], rdir, 'dir_cls_preds')):
        e = rel_err(got, ref)
        print('end to end', key, e, 'worst element / tol', assert_close(got, ref, key))
        assert e < TOL, (key, e)


@pytest.mark.parametrize('flip,aligned', [(False, True), (True, True), (False, False)])
def test_voxel_sample_vs_oracle(flip, aligned):
    """SURVEY.md row a8: the CUDA voxel_sample against the oracle (which equals the verbatim
    reference function, tests/test_oracle_golden.py)."""
    rng = np.random.RandomState(13)
    nx, ny, nz, c = 40, 32, 16, 6
    # smooth features so trilinear taps are not noise-amplifying; nearest mode uses the same
    vox = torch.cat([syn.smooth_field(rng, c, ny, nz, cell=4) for _ in range(nx)], 0)
    vox = vox.permute(1, 0, 2, 3)[None].contiguous()          # [1, C, Nx, Ny, Nz]
    vrange, vsize = [0.0, -8.0, -2.0, 20.0, 8.0, 2.0], [0.5, 0.5, 0.25]
    depths = torch.linspace(2.0, 18.0, 16)
    k = torch.tensor([[40., 0, 32, 0], [0, 40., 16, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    l2c = torch.tensor([[0., -1, 0, 0], [0, 0, -1, 0.3], [1, 0, 0, 0.1], [0, 0, 0, 1]])
    proj = k @ l2c
    args = (vrange, vsize, depths, proj, 4, torch.tensor([1.02, 0.98]),
            torch.tensor([1.0, 2.0]), flip, (32, 64), (30, 62))
    ref = O.voxel_sample(vox, *args, aligned=aligned)
    got = modules.voxel_sample(vox.cuda(), *args, aligned=aligned)
    assert got.shape == ref.shape == (1, c, 4, 8, 16)
    assert float(ref.abs().sum()) > 0
    if aligned:
        e = rel_err(got, ref)
        print('voxel_sample', flip, e)
        assert e < 1e-4
    else:
        # nearest: identical taps except where fp32 rounding of the coordinate sits on a tie
        bad = float(((got.cpu() - ref).abs().amax(1) > 1e-6).float().mean())
        print('voxel_sample nearest mismatching', bad)
        assert bad <= 0.02


@pytest.mark.parametrize('tpi', ['2', '5'])
@pytest.mark.parametrize('name', ['neck_dfm_mt', 'neck_imvoxel_mt'])
def test_neck_multitile_items_share_a_weight_image(name, tpi):
    """conv_tc_neck.cuh keeps the accumulators of several tiles in registers so that one weight image
    serves all of them (tiles-per-item, chosen from the grid size: 1 on these small fixtures).
    Forced here to 2 and 5 (capped per layer by NK_ACC_COLS / (Zo * NCTA) columns) on the 3 x 3-tile
    reference fixtures: same result as one tile per item."""
    gold = np.load(os.path.join(GOLDEN, name + '.npz'))
    rng, x = make_neck_mt_case(name)
    mod = (modules.DfMNeck(64, 256, num_frames=2) if name == 'neck_dfm_mt'
           else modules.OutdoorImVoxelNeck(64, 256))
    mod.load_state_dict(syn.make_neck_params(rng, mod.state_dict()), strict=True)
    mod = mod.cuda().eval()
    os.environ['DFM_NECK_TPI'] = tpi
    try:
        y = mod(x.cuda())[0]
        capi.sync_check()
    finally:
        os.environ.pop('DFM_NECK_TPI', None)
    e = rel_err(y, torch.from_numpy(gold['y']))
    print(name, 'tiles per item', tpi, e)
    assert e < TOL


@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_spp_unet_tail_vs_oracle_and_channels_last_backbone(impl):
    """SURVEY.md section 8(f) row 2: SPPUNetNeck.lastconv on CUDA against the oracle (equal to
    the verbatim reference module, tests/test_oracle_golden.py), and DfMBackbone fed by its
    channels-last twin against DfMBackbone fed by the NCHW tensor."""
    h, w, d = 64, 128, 8
    rng = np.random.RandomState(77)
    p = {'lastconv.0.conv.weight': torch.from_numpy(syn._kaiming(rng, (32, 32, 3, 3), 32 * 9)),
         'lastconv.0.gn.weight': torch.from_numpy((0.5 + rng.random_sample(32)).astype(np.float32)),
         'lastconv.0.gn.bias': torch.from_numpy((0.2 * rng.standard_normal(32)).astype(np.float32)),
         'lastconv.1.weight': torch.from_numpy(syn._kaiming(rng, (32, 32, 1, 1), 32))}
    tail = modules.SPPUNetNeckTail(conv_impl=impl)
    tail.load_state_dict(p, strict=True)
    tail = tail.cuda().eval()
    xc = syn.smooth_field(rng, 32, h, w)
    xp = syn.smooth_field(rng, 32, h, w)
    with torch.no_grad():
        rc, rp = O.spp_unet_lastconv(p, xc), O.spp_unet_lastconv(p, xp)
    cur, prev = tail(xc.cuda()), tail(xp.cuda())
    capi.sync_check()
    for got, ref in ((cur, rc), (prev, rp)):
        e = rel_err(got, ref)
        print('spp-unet tail', impl, e)
        assert e < (2e-5 if impl == 'simt' else 1e-4)
        assert torch.equal(got._dfm_cl.permute(2, 0, 1)[None], got)
    _, _, metas, params = syn.make_kitti_pair(78, h, w, d)
    cfg = syn.depth_cfg_for(d)
    bb = _backbone(params, cfg, 'auto')
    with torch.no_grad():
        a = bb(cur, prev, copy.deepcopy(metas))                  # channels-last twins
        b = bb(cur.clone(), prev.clone(), copy.deepcopy(metas))  # NCHW tensors (twin dropped)
    capi.sync_check()
    for x, y in zip(a, b):
        assert rel_err(x, y) < 1e-5
