"""Anchor3DHead forward (mmdet3d/models/dense_heads/anchor3d_head.py:139-164), the box head of
the MultiViewDfM (Waymo) configs: the mirror module, the C ABI, the 1x1-conv tensor-core kernel
(csrc/head1x1_tc.cuh) and its fp32 fall-back.

* CPU: the fp32 restatement below reproduces ``tests/golden/anchor3d_head.npz`` (written by
  ``tests/golden/make_anchor3d_golden.py`` from the verbatim reference methods; the inputs
  regenerate from ``synthetic.make_anchor3d_head_case``), the mirror has
  the reference ``state_dict``, both Waymo configs build it, checkpoints load into it, and the
  layer bound of the per-layer method (tests/layer_check.py) separates a lost bf16 term at K=256.
* GPU: fixture parity of both paths, an fp64 per-layer check (max-norm and element-wise on the
  cells beside every 128-cell tile seam and on the ragged tail), canary tails, repeatability,
  error paths, and Waymo box regressions end to end (lifting -> neck -> head) against the oracle.
"""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import depth_from_motion_b200 as pkg
from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import checkpoint as ck
from depth_from_motion_b200 import synthetic as syn
from tests.layer_check import SEPARATION, elementwise_errors, layer_bound, norm_errors, split16
from tests.util import GOLDEN, assert_close, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(GOLDEN, 'anchor3d_head.npz')
WAYMO_CONFIGS = ('multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py',
                 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py')
# the shipped head: 3 sizes x 2 rotations, 3 classes, sigmoid classification, 7-value box code
WAYMO_ANCHORS = dict(type='AlignedAnchor3DRangeGenerator',
                     ranges=[[-35.0, -75.0, 0, 75.0, 75.0, 0]] * 3,
                     sizes=[[0.91, 0.84, 1.74], [1.81, 0.84, 1.77], [4.73, 2.08, 1.77]],
                     rotations=[0, 1.57], reshape_out=False)
FLOOR_C = 8.0     # fp32 accumulation floor of the stage tests: 8 sqrt(K) 2^-24
TILE = 128        # cells per tile of head1x1_tc_kernel
ORDER = ('conv_cls', 'conv_dir_cls', 'conv_reg')   # row order of the combined GEMM


def anchor3d_head_forward(p, x):
    """fp32 restatement of Anchor3DHead.forward_single (anchor3d_head.py:159-164): the three
    1x1 convs with bias.  p: state dict, x [B, C, H, W] -> (cls_score, bbox_pred, dir or None)."""
    def conv(name):
        return F.conv2d(x, p[name + '.weight'], p[name + '.bias'])
    d = conv('conv_dir_cls') if 'conv_dir_cls.weight' in p else None
    return conv('conv_cls'), conv('conv_reg'), d


def load_fixture():
    """(fixture dict with the regenerated input under 'x', parameters).  Inputs regenerate from
    the seed; the stored checksums pin them to what the reference outputs were computed from."""
    g = dict(np.load(FIXTURE))
    x, params = syn.make_anchor3d_head_case(**syn.ANCHOR3D_HEAD_CASE)
    assert float(x.double().sum()) == pytest.approx(float(g['x_sum']), rel=1e-12)
    assert float(x.double().abs().sum()) == pytest.approx(float(g['x_abs']), rel=1e-12)
    assert sum(float(v.double().abs().sum()) for v in params.values()) == \
        pytest.approx(float(g['w_abs']), rel=1e-12)
    g['x'] = x.numpy()
    return g, params


def waymo_head(**kw):
    args = dict(num_classes=3, in_channels=256, feat_channels=256,
                anchor_generator=WAYMO_ANCHORS, bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'),
                loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25,
                              loss_weight=1.0))
    args.update(kw)
    return modules.Anchor3DHead(**args)


# ---------------------------------------------------------------------------------------------
# fp64 reference and the bf16-split emulation of the combined 1x1 GEMM
# ---------------------------------------------------------------------------------------------
def combined(p, dev):
    ws = [p[n + '.weight'] for n in ORDER if n + '.weight' in p]
    bs = [p[n + '.bias'] for n in ORDER if n + '.bias' in p]
    w = torch.cat([t.reshape(t.shape[0], -1) for t in ws]).to(dev)
    return w, torch.cat(bs).to(dev)


def gemm_reference(p, x):
    """x [1, K, H, W] -> fp64 (ref, 3-term split, x_lo dropped, w_lo dropped, product scale),
    each [N, H*W] with rows cls | dir | reg, bias included."""
    w, b = combined(p, x.device)
    k = x.shape[1]
    x2 = x[0].reshape(k, -1)
    b64 = b.double()[:, None]
    ref = w.double() @ x2.double() + b64
    xh, xl = split16(x2)
    wh, wl = split16(w)
    a = wh @ xh
    return (ref, a + wh @ xl + wl @ xh + b64, a + wl @ xh + b64, a + wh @ xl + b64,
            w.double().abs() @ x2.double().abs() + b64.abs())


def seam_cells(n):
    """Cells beside every 128-cell tile seam, the first and last cell, and the ragged tail."""
    s = {0, n - 1}
    for t in range(TILE, n, TILE):
        s.update((t - 1, t))
    s.update(range(n // TILE * TILE, n))
    return torch.tensor(sorted(s))


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
def test_oracle_reproduces_fixture():
    g, p = load_fixture()
    cls, box, dirc = anchor3d_head_forward(p, torch.from_numpy(g['x']))
    for got, key in ((cls, 'cls_score'), (box, 'bbox_pred'), (dirc, 'dir_cls_preds')):
        assert rel_err(got, g[key]) <= 1e-6, key


def test_mirror_state_dict_matches_reference():
    g, _ = load_fixture()
    m = waymo_head()
    assert [[k, ','.join(str(n) for n in v.shape)] for k, v in m.state_dict().items()] == \
        [[k, s] for k, s in zip(g['state_keys'].tolist(), g['state_shapes'].tolist())]
    assert (m.num_anchors, m.cls_out_channels, m.box_code_size) == (6, 18, 7)


@pytest.mark.parametrize('cfg_name', WAYMO_CONFIGS)
def test_waymo_configs_build_anchor3d_head(cfg_name):
    """bbox_head_3d of both shipped Waymo configs, with train_cfg / test_cfg injected as
    detectors/dfm.py:104-105 does."""
    with open(os.path.join(GOLDEN, 'reference_io.json')) as f:
        model = json.load(f)['configs'][cfg_name]
    cfg = dict(model['bbox_head_3d'])
    cfg.update(train_cfg=model['train_cfg'], test_cfg=model['test_cfg'])
    hd = pkg.build_head(cfg)
    assert isinstance(hd, modules.Anchor3DHead)
    assert hd.num_anchors == 6 and hd.num_classes == 3
    assert (hd.conv_cls.out_channels, hd.conv_reg.out_channels,
            hd.conv_dir_cls.out_channels) == (18, 42, 12)
    assert hd.conv_cls.kernel_size == (1, 1) and hd.conv_cls.in_channels == 256
    assert hd.test_cfg['nms_thr'] == model['test_cfg']['nms_thr']
    cfg.update(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
               use_direction_classifier=False)
    hd = pkg.build_head(cfg)
    assert hd.num_classes == 4 and hd.cls_out_channels == 24
    assert not hasattr(hd, 'conv_dir_cls')
    assert not any(k.startswith('conv_dir_cls') for k in hd.state_dict())


def test_load_hot_path_loads_bbox_head_3d():
    _, p = load_fixture()
    det = {'bbox_head_3d.' + k: v for k, v in p.items()}
    det['neck_3d.model.0.conv.weight'] = torch.zeros(3)
    m = waymo_head()
    ck.load_hot_path({'state_dict': det}, head=m, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in p.items())
    with pytest.raises(KeyError):
        ck.load_hot_path({'state_dict': {'neck_3d.x': torch.zeros(1)}}, head=waymo_head())


def test_bound_separates_lost_term_cpu():
    """On the oracle inputs at K = 256 the layer bound max(6 e3, 8 sqrt(K) 2^-24) stays at
    least SEPARATION times below e2, the error with one bf16 lo term dropped: a kernel that
    loses a term cannot pass the GPU check."""
    g, p = load_fixture()
    ref, y3, y2x, y2w, scale = gemm_reference(p, torch.from_numpy(g['x']))
    e3, e2 = norm_errors((y3, y2x, y2w), ref)
    bound = layer_bound(e3, 256, FLOOR_C)
    assert SEPARATION * bound <= e2, (e3, e2, bound)
    cells = seam_cells(ref.shape[1])
    _, _, e2_ew, b_ew = elementwise_errors(y3[:, cells], ref[:, cells], y3[:, cells],
                                           y2x[:, cells], y2w[:, cells], scale[:, cells], 256,
                                           FLOOR_C)
    assert SEPARATION * b_ew <= e2_ew


def test_anchor3d_desc_matches_the_c_header(tmp_path):
    cname, cls = 'dfm_anchor3d_head_desc_t', capi.Anchor3DHeadDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>',
             f'#include "{os.path.join(ROOT, "include", "dfm_b200.h")}"', 'int main(void) {',
             f'printf("size %zu\\n", sizeof({cname}));']
    lines += [f'printf("{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in cls._fields_]
    src = tmp_path / 'abi.c'
    src.write_text('\n'.join(lines + ['return 0;', '}']))
    exe = tmp_path / 'abi'
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-o', str(exe), str(src)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                 check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _cuda_head(p, impl='auto', **kw):
    m = waymo_head(conv_impl=impl, **kw)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _as_rows(outs):
    """(cls, box, dir) of one sample -> [N, H*W] rows cls | dir | reg"""
    cls, box, dirc = (t[0] if t is not None else None for t in outs)
    parts = [cls, dirc, box] if dirc is not None else [cls, box]
    return torch.cat([t.reshape(t.shape[0], -1) for t in parts]).double()


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_fixture_parity(impl):
    g, p = load_fixture()
    m = _cuda_head(p, impl)
    x = torch.from_numpy(g['x']).cuda()
    with torch.no_grad():
        m([x])
        capi.sync_check()
        _, tc0 = capi.launch_counters()
        cls, box, dirc = m([x])
        capi.sync_check()
        _, tc1 = capi.launch_counters()
    assert (tc1 > tc0) == (impl == 'auto'), (impl, tc0, tc1)
    for got, key in ((cls[0], 'cls_score'), (box[0], 'bbox_pred'), (dirc[0], 'dir_cls_preds')):
        e = rel_err(got, g[key])
        print('anchor3d_head fixture', impl, key, e, assert_close(got, g[key], key))
        assert e < 1e-3


def _bev_input(name):
    """(x [1, 256, H, W] on the GPU, state dict)"""
    g, p = load_fixture()
    if name == 'fixture':
        return torch.from_numpy(g['x']).cuda(), p
    rng = np.random.RandomState(303)
    if name == 'small':
        x = rng.standard_normal((1, 256, 5, 3))
    elif name == 'random_sign':
        x = rng.standard_normal((1, 256, 300, 220))
    else:
        # the benchmark's Waymo path: synthetic sample -> lifting -> DfMNeck -> BEV map
        from tests.test_stage_layers import make_neck_case
        mod, vol, _ = make_neck_case('waymo_dfm')
        with torch.no_grad():
            x = mod(vol)[0]
        capi.sync_check()
        assert tuple(x.shape) == (1, 256, 300, 220)
        return x.contiguous(), p
    return torch.from_numpy(x.astype(np.float32)).cuda(), p


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['fixture', 'waymo_neck', 'random_sign', 'small'])
def test_layer_vs_fp64(name):
    """The tensor-core GEMM against fp64: max-norm error <= max(6 e3, 8 sqrt(K) 2^-24) with that
    bound SEPARATION times below e2, and the element-wise form of it (scaled by the product
    scale sum |x||w| + |b|) on every tile-seam cell and the ragged tail."""
    x, p = _bev_input(name)
    m = _cuda_head(p)
    with torch.no_grad():
        m([x])
        capi.sync_check()
        capi.profile_report()
        capi.profile_enable(True)
        try:
            outs = m.forward_single(x)
            capi.sync_check()
            report = capi.profile_report()
        finally:
            capi.profile_enable(False)
    assert any(k.startswith('head1x1_tc<256->72>') for k in report), report
    got = _as_rows(outs)
    ref, y3, y2x, y2w, scale = gemm_reference({k: v.cuda() for k, v in p.items()}, x)
    e = float((got - ref).abs().max()) / float(ref.abs().max())
    e3, e2 = norm_errors((y3, y2x, y2w), ref)
    bound = layer_bound(e3, 256, FLOOR_C)
    print(f'anchor3d_head {name}: err {e:.3g} e3 {e3:.3g} bound {bound:.3g} e2 {e2:.3g}')
    assert e <= bound and SEPARATION * bound <= e2, (e, e3, bound, e2)
    cells = seam_cells(ref.shape[1]).to(ref.device)
    sel = [t[:, cells] for t in (got, ref, y3, y2x, y2w, scale)]
    g_ew, e3_ew, e2_ew, b_ew = elementwise_errors(*sel, 256, FLOOR_C)
    print(f'  seams/tail: gpu {g_ew:.3g} e3 {e3_ew:.3g} bound {b_ew:.3g} e2 {e2_ew:.3g}')
    assert g_ew <= b_ew and SEPARATION * b_ew <= e2_ew


class _RawHead:
    """The C handle driven directly, for caller-allocated output buffers."""

    def __init__(self, p, feat, nc, nr, nd, ny, nx, impl):
        L = capi.lib()
        desc = capi.Anchor3DHeadDesc(feat, nc, nr, nd, ny, nx, modules._IMPL[impl])
        self.h = ctypes.c_void_p()
        capi.check(L.dfm_anchor3d_head_create(ctypes.byref(desc), ctypes.byref(self.h)),
                   'create')
        self.host = {}
        for k, v in p.items():
            self.host[k] = v.detach().float().contiguous().cpu()
            self.set(k, self.host[k])

    def set(self, k, v, numel=None):
        return capi.lib().dfm_anchor3d_head_set_param(
            self.h, k.encode(), ctypes.c_void_p(v.data_ptr()), v.numel() if numel is None else numel)

    def forward(self, x, cls, box, dirc):
        return capi.lib().dfm_anchor3d_head_forward(
            self.h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(cls.data_ptr()),
            ctypes.c_void_p(box.data_ptr()),
            ctypes.c_void_p(dirc.data_ptr()) if dirc is not None else None,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

    def close(self):
        capi.lib().dfm_anchor3d_head_destroy(self.h)


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['auto', 'simt'])
def test_no_overrun_repeatable_side_effect_free(impl):
    g, p = load_fixture()
    x = torch.from_numpy(g['x']).cuda()
    x0 = x.clone()
    ny, nx = x.shape[2:]
    hw, canary, tail = ny * nx, -12345.5, 1000
    h = _RawHead(p, 256, 18, 42, 12, ny, nx, impl)
    try:
        runs = []
        for _ in range(2):
            bufs = [torch.full((c * hw + tail,), canary, device='cuda') for c in (18, 42, 12)]
            assert h.forward(x, *bufs) == 0, capi.lib().dfm_last_error()
            capi.sync_check()
            for b in bufs:
                assert bool((b[-tail:] == canary).all()), 'write past the end of an output'
            runs.append([b[:-tail].clone() for b in bufs])
    finally:
        h.close()
    assert torch.equal(x, x0), 'the forward modified its input'
    for a, b in zip(*runs):
        assert torch.equal(a, b), 'two forwards differ'
    for got, key, c in zip(runs[0], ('cls_score', 'bbox_pred', 'dir_cls_preds'), (18, 42, 12)):
        assert rel_err(got.view(1, c, ny, nx), g[key]) < 1e-3, key


@pytest.mark.gpu
def test_errors():
    g, p = load_fixture()
    m = _cuda_head(p)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match='CUDA tensor'):
            m([torch.from_numpy(g['x'])])
        with pytest.raises(RuntimeError, match='channels'):
            m([torch.zeros((1, 128, 5, 3), device='cuda')])
    # missing parameters, wrong element counts, unknown keys (C ABI)
    h = _RawHead({k: v for k, v in p.items() if not k.startswith('conv_reg')}, 256, 18, 42, 12,
                 5, 3, 'auto')
    try:
        assert capi.lib().dfm_anchor3d_head_missing_params(h.h) == 2
        x = torch.zeros((1, 256, 5, 3), device='cuda')
        bufs = [torch.zeros(c * 15, device='cuda') for c in (18, 42, 12)]
        assert h.forward(x, *bufs) == 3                                  # DFM_ERR_STATE
        assert h.set('conv_reg.weight', p['conv_reg.weight'], 41 * 256) == 1   # DFM_ERR_INVALID
        assert h.set('conv_reg.bias', p['conv_reg.bias'], 43) == 1
        assert h.set('conv_bogus.weight', p['conv_reg.bias']) == 1
        assert h.set('conv_reg.weight', p['conv_reg.weight'].contiguous()) == 0
        assert h.set('conv_reg.bias', p['conv_reg.bias'].contiguous()) == 0
        assert capi.lib().dfm_anchor3d_head_missing_params(h.h) == 0
        assert h.forward(x, *bufs) == 0
        capi.sync_check()
    finally:
        h.close()
    # conv_impl='tc' on a feat_channels the tensor-core kernel does not take fails at create
    odd = waymo_head(feat_channels=24, conv_impl='tc').cuda().eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match='no tensor-core kernel'):
        odd([torch.zeros((1, 24, 5, 3), device='cuda')])


@pytest.mark.gpu
def test_auto_falls_back_on_wide_heads():
    """240 output channels exceed the widest tensor-core instantiation: 'auto' runs the fp32
    CUDA-core conv (no tensor-core launch), 'tc' refuses."""
    anchors = dict(WAYMO_ANCHORS, sizes=[[1.0, 1.0, 1.0]] * 10)
    rng = np.random.RandomState(7)
    m = waymo_head(feat_channels=128, anchor_generator=anchors)
    sd = {k: torch.from_numpy((rng.standard_normal(v.shape) * 0.1).astype(np.float32))
          for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    m = m.cuda().eval()
    x = torch.from_numpy(rng.standard_normal((1, 128, 19, 23)).astype(np.float32)).cuda()
    with torch.no_grad():
        m([x])
        capi.sync_check()
        _, tc0 = capi.launch_counters()
        cls, box, dirc = m([x])
        capi.sync_check()
        _, tc1 = capi.launch_counters()
    assert tc1 == tc0
    ref = anchor3d_head_forward({k: v.cuda().double() for k, v in sd.items()}, x.double())
    for got, r in zip((cls[0], box[0], dirc[0]), ref):
        assert rel_err(got, r) < 1e-5
    tc = waymo_head(feat_channels=128, anchor_generator=anchors, conv_impl='tc').cuda().eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match='no tensor-core kernel'):
        tc([x])


@pytest.mark.gpu
@pytest.mark.parametrize('t,agg,neck', [(1, 'mean', 'imvoxel'), (2, 'concat', 'dfm')])
def test_waymo_box_regressions_end_to_end(t, agg, neck):
    """All-CUDA MultiViewDfM segment (detectors/multiview_dfm.py:119-268, 321-326): lifting ->
    neck_3d -> Anchor3DHead against the all-oracle chain, on the grid of
    test_multiview_feature_transformation_mixin_vs_oracle (20 x 18 cells: two full tiles and a
    ragged one), for a batch of two samples with different metas."""
    from oracle import dfm_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    nv = 3
    n_voxels, vrange = [20, 18, 12], [0.0, -9.0, -2.0, 20.0, 9.0, 4.0]
    rng = np.random.RandomState(61)
    mod = (modules.DfMNeck(64, 256, num_frames=2) if neck == 'dfm'
           else modules.OutdoorImVoxelNeck(64, 256))
    sd = syn.make_neck_params(rng, mod.state_dict())
    mod.load_state_dict(sd, strict=True)
    mod = mod.cuda().eval()
    _, hp = load_fixture()
    head = _cuda_head(hp)

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
    with torch.no_grad():
        bev = host.feature_transformation(torch.stack(feats).cuda(), metas, nv, t)[0]
        cls, box, dirc = head([bev])                               # multiview_dfm.py:321-326
    capi.sync_check()
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
            rbev = (O.dfm_neck_forward(sd, vol, 64) if neck == 'dfm'
                    else O.imvoxel_neck_forward(sd, vol))[0]
            rcls, rbox, rdir = anchor3d_head_forward(hp, rbev)
        for got, ref, key in ((cls[0][b], rcls[0], 'cls_score'), (box[0][b], rbox[0], 'bbox_pred'),
                              (dirc[0][b], rdir[0], 'dir_cls_preds')):
            e = rel_err(got, ref)
            print('waymo end to end', neck, b, key, e, 'worst element / tol',
                  assert_close(got, ref, key))
            assert e < 1e-3, (key, e)
