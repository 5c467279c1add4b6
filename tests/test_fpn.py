"""mmdet's FPN as the image neck of both MultiViewDfM (Waymo) configs: the mirror module, the C
ABI, the lateral tensor-core kernel with the fused top-down merge (csrc/fpn_kernels.cuh), the
3x3 fpn_convs on the 2-D layer driver, and the fp32 CUDA-core path.

mmdet is not part of the reference tree, so ``fpn_forward`` below restates mmdet 2.24's
``FPN.forward`` for the configuration both Waymo configs use (start_level 0, no extra convs, no
norm or activation, nearest upsampling to the finer level's size); no verbatim source is
available to execute.

* CPU: ``state_dict`` layout, both Waymo configs through the local registry, the rejected
  options, checkpoint loading, the descriptor ABI, the restatement against an ``nn.Conv2d`` fp32
  build and the nearest index rule, and the bound separation of every new layer class.
* GPU: the whole module against fp64 for auto and simt (cases A, B, C below), every layer
  against fp64 from the GPU's own inputs (max-norm and element-wise on the tile seams, image
  boundaries and ragged tails), canary tails, repeatability, error paths, the auto fall-back,
  and FPN -> lifting -> 3-D neck -> Anchor3DHead end to end against the all-oracle chain.
"""
import ctypes
import json
import math
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
from tests.layer_check import (SEPARATION, conv_planes, elementwise_errors, emulated_outputs,
                               layer_bound, norm_errors, product_scale, split16)
from tests.util import GOLDEN, assert_close, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WAYMO_CONFIGS = ('multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py',
                 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py')
IN_CH = [256, 512, 1024, 2048]
FLOOR_C = 8.0     # fp32 accumulation floor of the layer bound: 8 sqrt(K) 2^-24
TILE = 128        # cells per tile of fpn_lateral_tc_kernel
# (input image H, W, images per call): A the shipped pyramid of 5 views, B a ragged pyramid
# (non-2x nearest ratios), C coarse levels smaller than one tile
CASES = {'A': (832, 1248, 5), 'B': (300, 452, 2), 'C': (64, 96, 1)}


def levels(h, w):
    """C2..C5 sizes of a ResNet on an h x w image (every stride-2 stage rounds up)."""
    out = []
    for s in range(5):
        h, w = -(-h // 2), -(-w // 2)
        if s >= 1:
            out.append((h, w))
    return out


def fpn_forward(p, xs):
    """fp64-capable restatement of mmdet 2.24 ``FPN.forward`` (mmdet/models/necks/fpn.py) for
    start_level 0, add_extra_convs False, num_outs == len(inputs), no norm / activation and
    upsample_cfg dict(mode='nearest'); no verbatim source is available to execute.
    p: state dict, xs: 4 NCHW maps -> tuple of 4 NCHW maps."""
    lat = [F.conv2d(x, p[f'lateral_convs.{i}.conv.weight'], p[f'lateral_convs.{i}.conv.bias'])
           for i, x in enumerate(xs)]
    for i in range(len(lat) - 1, 0, -1):                  # top-down pathway
        lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], size=lat[i - 1].shape[2:],
                                                mode='nearest')
    return tuple(F.conv2d(l, p[f'fpn_convs.{i}.conv.weight'], p[f'fpn_convs.{i}.conv.bias'],
                          padding=1) for i, l in enumerate(lat))


def nearest_index(dst, n_in, n_out):
    """PyTorch's legacy nearest rule for F.interpolate(size=...)."""
    if n_in == n_out:
        return dst
    if n_out == 2 * n_in:
        return dst >> 1
    scale = np.float32(n_in) / np.float32(n_out)
    return min(int(np.floor(np.float32(dst) * scale)), n_in - 1)


def make_params(seed, out_channels=64, in_channels=IN_CH):
    g = torch.Generator().manual_seed(seed)
    p = {}
    for i, c in enumerate(in_channels):
        p[f'lateral_convs.{i}.conv.weight'] = torch.randn(out_channels, c, 1, 1, generator=g) / math.sqrt(c)
        p[f'lateral_convs.{i}.conv.bias'] = 0.1 * torch.randn(out_channels, generator=g)
        k = 9 * out_channels
        p[f'fpn_convs.{i}.conv.weight'] = torch.randn(out_channels, out_channels, 3, 3,
                                                      generator=g) / math.sqrt(k)
        p[f'fpn_convs.{i}.conv.bias'] = 0.1 * torch.randn(out_channels, generator=g)
    return p


def make_inputs(seed, h, w, n, device='cpu', in_channels=IN_CH):
    """Non-negative (post-ReLU) pyramid features C2..C5 of n images of size h x w."""
    g = torch.Generator(device=device).manual_seed(seed)
    return [torch.randn((n, c) + s, generator=g, device=device).abs_()
            for c, s in zip(in_channels, levels(h, w))]


def waymo_fpn(**kw):
    args = dict(in_channels=IN_CH, out_channels=64, num_outs=4)
    args.update(kw)
    return modules.FPN(**args)


def lateral_reference(p, x, i):
    """x [N, K, h, w] -> fp64 (W x + b, 3-term split, x_lo dropped, w_lo dropped, product
    scale), each [C, N*h*w] (cells of all images, image-major)."""
    w = p[f'lateral_convs.{i}.conv.weight'].to(x.device)
    b = p[f'lateral_convs.{i}.conv.bias'].to(x.device).double()[:, None]
    w = w.reshape(w.shape[0], -1)
    x2 = x.transpose(0, 1).reshape(x.shape[1], -1)
    xh, xl = split16(x2)
    wh, wl = split16(w)
    a = wh @ xh
    return (w.double() @ x2.double() + b, a + wh @ xl + wl @ xh + b, a + wl @ xh + b,
            a + wh @ xl + b, w.double().abs() @ x2.double().abs() + b.abs())


def lateral_cells(n, hw):
    """Columns (image-major cells) beside every 128-cell tile seam of each image, each image's
    first and last cell (the image boundaries of the batched launch) and its ragged tail."""
    s = set()
    for i in range(n):
        o = i * hw
        s.update((o, o + hw - 1))
        for t in range(TILE, hw, TILE):
            s.update((o + t - 1, o + t))
        s.update(range(o + hw // TILE * TILE, o + hw))
    return torch.tensor(sorted(s))


def conv_seam_mask(h, w):
    """Cells on both sides of every 16 x 8 tile seam of the 2-D conv (either orientation) and
    on the map's edges."""
    ys, xs = torch.arange(h), torch.arange(w)
    my = (ys % 8 == 0) | (ys % 8 == 7) | (ys == h - 1)
    mx = (xs % 8 == 0) | (xs % 8 == 7) | (xs == w - 1)
    return my[:, None] | mx[None, :]


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
def test_state_dict_layout():
    m = waymo_fpn()
    sd = m.state_dict()
    want = {}
    for i, c in enumerate(IN_CH):
        want[f'lateral_convs.{i}.conv.weight'] = (64, c, 1, 1)
        want[f'lateral_convs.{i}.conv.bias'] = (64,)
    for i in range(4):
        want[f'fpn_convs.{i}.conv.weight'] = (64, 64, 3, 3)
        want[f'fpn_convs.{i}.conv.bias'] = (64,)
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert len(sd) == 16


@pytest.mark.parametrize('cfg_name', WAYMO_CONFIGS)
def test_waymo_configs_build_fpn(cfg_name):
    with open(os.path.join(GOLDEN, 'reference_io.json')) as f:
        cfg = json.load(f)['configs'][cfg_name]['neck']
    m = pkg.build_neck(dict(cfg))
    assert isinstance(m, modules.FPN)
    assert (m.in_channels, m.out_channels, m.num_outs) == (IN_CH, 64, 4)


def test_unsupported_options_raise():
    with open(os.path.join(GOLDEN, 'reference_io.json')) as f:
        kitti = json.load(f)['configs']['dfm_r34_1x8_kitti-3d-3class.py']['neck_2d']
    with pytest.raises(NotImplementedError):
        pkg.build_neck(dict(kitti))
    for kw in (dict(add_extra_convs='on_output'), dict(add_extra_convs=True), dict(num_outs=5),
               dict(norm_cfg=dict(type='BN')), dict(act_cfg=dict(type='ReLU')),
               dict(conv_cfg=dict(type='Conv2d')), dict(upsample_cfg=dict(mode='bilinear')),
               dict(upsample_cfg=dict(scale_factor=2)), dict(start_level=1),
               dict(in_channels=[256, 512, 1024, 2040]), dict(out_channels=56),
               dict(in_channels=[256, 512, 1024])):
        with pytest.raises(NotImplementedError):
            waymo_fpn(**kw)
    with pytest.raises(ValueError):
        waymo_fpn(num_outs=3)


def test_load_hot_path_loads_fpn():
    p = make_params(5)
    det = {'neck.' + k: v for k, v in p.items()}
    det['neck_3d.model.0.conv.weight'] = torch.zeros(3)
    det['backbone.conv1.weight'] = torch.zeros(3)
    m = waymo_fpn()
    ck.load_hot_path({'state_dict': det}, img_neck=m, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in p.items())


def test_fpn_desc_matches_the_c_header(tmp_path):
    cname, cls = 'dfm_fpn_desc_t', capi.FpnDesc
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


def test_nearest_rule_matches_interpolate():
    """The index rule the kernels implement selects what F.interpolate(size=) selects, on the
    ragged pyramid of case B (75 -> 38 -> 19 -> 10 rows, 113 -> 57 -> 29 -> 15 columns)."""
    sizes = levels(300, 452)
    for (hf, wf), (hc, wc) in zip(sizes[:-1], sizes[1:]):
        for n_in, n_out in ((hc, hf), (wc, wf)):
            for dt in (torch.float32, torch.float64):
                src = torch.arange(n_in, dtype=dt)[None, None, :, None]
                got = F.interpolate(src, size=(n_out, 1), mode='nearest')[0, 0, :, 0]
                want = [nearest_index(d, n_in, n_out) for d in range(n_out)]
                assert got.long().tolist() == want, (n_in, n_out, dt)
    assert nearest_index(5, 19, 38) == 2 and nearest_index(37, 19, 38) == 18


def test_restatement_matches_conv2d_build():
    """The fp64 restatement against the mirror's own nn.Conv2d containers run in fp32 with
    F.interpolate, on the ragged pyramid of case B (one image)."""
    p = make_params(11)
    m = waymo_fpn()
    m.load_state_dict(p, strict=True)
    xs = make_inputs(12, 300, 452, 1)
    with torch.no_grad():
        lat = [c.conv(x) for c, x in zip(m.lateral_convs, xs)]
        for i in range(3, 0, -1):
            lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], size=lat[i - 1].shape[2:])
        f32 = [c.conv(x) for c, x in zip(m.fpn_convs, lat)]
        f64 = fpn_forward({k: v.double() for k, v in p.items()}, [x.double() for x in xs])
    for a, b in zip(f32, f64):
        assert a.shape == b.shape
        assert rel_err(a, b) < 2e-6


def test_bound_separates_lost_term_cpu():
    """For every new layer class -- the laterals at K = 256, 512, 1024, 2048 and the fpn_convs
    at K = 576 -- the bound max(6 e3, 8 sqrt(K) 2^-24) stays SEPARATION times below e2 (one bf16
    lo term dropped), on case C's inputs (max-norm and element-wise)."""
    h, w, n = CASES['C']
    p = make_params(21)
    xs = make_inputs(22, h, w, n)
    with torch.no_grad():
        lat = [None] * 4
        for i in range(3, -1, -1):
            k = IN_CH[i]
            ref, y3, y2x, y2w, scale = lateral_reference(p, xs[i], i)
            e3, e2 = norm_errors((y3, y2x, y2w), ref)
            bound = layer_bound(e3, k, FLOOR_C)
            assert SEPARATION * bound <= e2, ('lateral', k, e3, e2, bound)
            cells = lateral_cells(n, xs[i].shape[2] * xs[i].shape[3])
            _, _, e2_ew, b_ew = elementwise_errors(
                y3[:, cells], ref[:, cells], y3[:, cells], y2x[:, cells], y2w[:, cells],
                scale[:, cells], k, FLOOR_C)
            assert SEPARATION * b_ew <= e2_ew, ('lateral elementwise', k)
            lat[i] = ref.float().reshape(64, n, *xs[i].shape[2:]).transpose(0, 1)
            if i < 3:
                lat[i] = lat[i] + F.interpolate(lat[i + 1], size=lat[i].shape[2:])
        for i in range(4):
            wgt = p[f'fpn_convs.{i}.conv.weight']
            x = lat[i][:1]
            ref = conv_planes(x.double(), wgt.double())
            ys = emulated_outputs(x, wgt)
            e3, e2 = norm_errors(ys, ref)
            bound = layer_bound(e3, 576, FLOOR_C)
            assert SEPARATION * bound <= e2, ('fpn_conv', i, e3, e2, bound)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _cuda_fpn(p, impl='auto', **kw):
    m = waymo_fpn(conv_impl=impl, **kw)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _profiled(fn):
    capi.sync_check()
    capi.profile_report()
    capi.profile_enable(True)
    try:
        out = fn()
        capi.sync_check()
        return out, capi.profile_report()
    finally:
        capi.profile_enable(False)


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['auto', 'simt'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_module_vs_fp64(case, impl):
    """All four outputs against the fp64 restatement within the 1e-3 bars; only 'auto' launches
    tensor-core kernels."""
    h, w, n = CASES[case]
    p = make_params(31)
    xs = make_inputs(32, h, w, n, device='cuda')
    m = _cuda_fpn(p, impl)
    with torch.no_grad():
        m(xs)
        capi.sync_check()
        _, tc0 = capi.launch_counters()
        outs = m(xs)
        capi.sync_check()
        _, tc1 = capi.launch_counters()
        ref = fpn_forward({k: v.cuda().double() for k, v in p.items()}, [x.double() for x in xs])
    assert (tc1 > tc0) == (impl == 'auto'), (impl, tc0, tc1)
    if impl == 'auto':
        assert tc1 - tc0 == 4 + 4 * n      # 4 lateral GEMMs, one fpn_conv per level and image
    for l, (got, r) in enumerate(zip(outs, ref)):
        assert got.shape == r.shape
        e = rel_err(got, r)
        print(f'fpn {case} {impl} out[{l}] rel {e:.3g} worst/tol {assert_close(got, r, str(l)):.3g}')
        assert e < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CASES))
def test_layers_vs_fp64(case):
    """Each merged_l against fp64 from the GPU's own merged_{l+1} (error over max|W x + b|),
    each fpn_conv against fp64 from the GPU's merged_l, held to max(6 e3, 8 sqrt(K) 2^-24) with
    e2 SEPARATION times above, in max-norm and element-wise on the tile seams, image boundaries
    and ragged tails.  Every tensor-core class launched is compared."""
    h, w, n = CASES[case]
    p = make_params(41)
    pc = {k: v.cuda() for k, v in p.items()}
    xs = make_inputs(42, h, w, n, device='cuda')
    m = _cuda_fpn(p)
    with torch.no_grad():
        m(xs)
        _, report = _profiled(lambda: m(xs))
    sizes = levels(h, w)
    for k in IN_CH:
        assert any(c.startswith(f'fpn_lateral_tc<{k}->64>') for c in report), report
    assert any(c.startswith('conv2d_tc<64->64,s1') for c in report), report
    merged = [m.debug_tensor(f'merged{l}', (n,) + sizes[l] + (64,)) for l in range(4)]
    raw = [m.debug_tensor(f'fpn{l}', (n,) + sizes[l] + (64,)) for l in range(4)]
    worst = []
    with torch.no_grad():
        for l in range(4):
            k, (hl, wl) = IN_CH[l], sizes[l]
            ref, y3, y2x, y2w, scale = lateral_reference(pc, xs[l], l)
            if l < 3:
                up = F.interpolate(merged[l + 1].permute(0, 3, 1, 2), size=(hl, wl))
                up = up.double().transpose(0, 1).reshape(64, -1)
            else:
                up = torch.zeros_like(ref)
            got = merged[l].permute(3, 0, 1, 2).reshape(64, -1).double() - up
            e = float((got - ref).abs().max()) / float(ref.abs().max())
            e3, e2 = norm_errors((y3, y2x, y2w), ref)
            bound = layer_bound(e3, k, FLOOR_C)
            print(f'fpn {case} lateral K={k}: err {e:.3g} e3 {e3:.3g} bound {bound:.3g} '
                  f'e2 {e2:.3g}')
            assert e <= bound and SEPARATION * bound <= e2, (l, e, e3, bound, e2)
            worst.append(e / e3)
            cells = lateral_cells(n, hl * wl).to(ref.device)
            sel = [t[:, cells] for t in (got, ref, y3, y2x, y2w, scale)]
            g_ew, e3_ew, e2_ew, b_ew = elementwise_errors(*sel, k, FLOOR_C)
            print(f'  seams/tails: gpu {g_ew:.3g} e3 {e3_ew:.3g} bound {b_ew:.3g} e2 {e2_ew:.3g}')
            assert g_ew <= b_ew and SEPARATION * b_ew <= e2_ew, l
            del ref, y3, y2x, y2w, scale, up, got
            wgt = pc[f'fpn_convs.{l}.conv.weight']
            mask = conv_seam_mask(hl, wl).to(wgt.device)
            for i in range(n):
                x = merged[l][i].permute(2, 0, 1)[None]
                ref = conv_planes(x.double(), wgt.double())
                ys = emulated_outputs(x, wgt)
                gotc = raw[l][i].permute(2, 0, 1)[None].double()
                e = float((gotc - ref).abs().max()) / float(ref.abs().max())
                e3, e2 = norm_errors(ys, ref)
                bound = layer_bound(e3, 576, FLOOR_C)
                assert e <= bound and SEPARATION * bound <= e2, ('fpn_conv', l, i, e, e3, e2)
                worst.append(e / e3)
                sel = [t[0][:, mask] for t in (gotc, ref) + tuple(ys) +
                       (product_scale(x.double(), wgt.double()),)]
                g_ew, _, e2_ew, b_ew = elementwise_errors(*sel, 576, FLOOR_C)
                assert g_ew <= b_ew and SEPARATION * b_ew <= e2_ew, ('fpn_conv seams', l, i)
            print(f'fpn {case} fpn_conv {l}: last image err {e:.3g} e3 {e3:.3g} e2 {e2:.3g}')
    print(f'fpn {case}: worst err / e3 {max(worst):.3g}')


class _RawFpn:
    """The C handle driven directly, for caller-allocated buffers."""

    def __init__(self, p, h, w, n, impl, out_channels=64, skip=()):
        L = capi.lib()
        sizes = levels(h, w)
        d = capi.FpnDesc()
        d.in_channels[:] = IN_CH
        d.out_channels = out_channels
        d.level_h[:] = [s[0] for s in sizes]
        d.level_w[:] = [s[1] for s in sizes]
        d.num_images, d.conv_impl = n, modules._IMPL[impl]
        self.h = ctypes.c_void_p()
        capi.check(L.dfm_fpn_create(ctypes.byref(d), ctypes.byref(self.h)), 'create')
        self.host = {k: v.detach().float().contiguous().cpu() for k, v in p.items()}
        for k, v in self.host.items():
            if k not in skip:
                assert self.set(k, v) == 0

    def set(self, k, v, numel=None):
        return capi.lib().dfm_fpn_set_param(self.h, k.encode(), ctypes.c_void_p(v.data_ptr()),
                                            v.numel() if numel is None else numel)

    def forward(self, xs, outs):
        arr = ctypes.c_void_p * 4
        return capi.lib().dfm_fpn_forward(
            self.h, arr(*[x.data_ptr() for x in xs]), arr(*[o.data_ptr() for o in outs]),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

    def debug(self, name, numel):
        out = torch.empty(max(numel, 1), device='cuda')
        return capi.lib().dfm_fpn_debug_tensor(self.h, name.encode(), ctypes.c_void_p(
            out.data_ptr()), numel, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

    def close(self):
        capi.lib().dfm_fpn_destroy(self.h)


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['auto', 'simt'])
def test_no_overrun_repeatable_side_effect_free(impl):
    h, w, n = CASES['B']
    p = make_params(51)
    xs = make_inputs(52, h, w, n, device='cuda')
    x0 = [x.clone() for x in xs]
    sizes = levels(h, w)
    canary, tail = -12345.5, 1000
    f = _RawFpn(p, h, w, n, impl)
    try:
        runs = []
        for _ in range(2):
            bufs = [torch.full((n * 64 * a * b + tail,), canary, device='cuda') for a, b in sizes]
            assert f.forward(xs, bufs) == 0, capi.lib().dfm_last_error()
            capi.sync_check()
            for b in bufs:
                assert bool((b[-tail:] == canary).all()), 'write past the end of an output'
            runs.append([b[:-tail].clone() for b in bufs])
    finally:
        f.close()
    assert all(torch.equal(a, b) for a, b in zip(xs, x0)), 'the forward modified its input'
    for a, b in zip(*runs):
        assert torch.equal(a, b), 'two forwards differ'
    ref = fpn_forward({k: v.cuda().double() for k, v in p.items()}, [x.double() for x in xs])
    for got, r in zip(runs[0], ref):
        assert rel_err(got.view(r.shape), r) < 1e-3


@pytest.mark.gpu
def test_errors():
    h, w, n = CASES['C']
    p = make_params(61)
    xs = make_inputs(62, h, w, n, device='cuda')
    m = _cuda_fpn(p)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match='CUDA tensor'):
            m([x.cpu() for x in xs])
        with pytest.raises(ValueError):
            m(xs[:3])
        with pytest.raises(ValueError):                  # channel count
            m([xs[0][:, :128]] + xs[1:])
        with pytest.raises(ValueError):                  # batch sizes disagree
            m([torch.cat([xs[0], xs[0]])] + xs[1:])
    m.train()
    with pytest.raises(RuntimeError, match='forward-only'):
        m(xs)
    sizes = levels(h, w)
    skip = ('fpn_convs.2.conv.bias', 'lateral_convs.3.conv.weight')
    f = _RawFpn(p, h, w, n, 'auto', skip=skip)
    try:
        L = capi.lib()
        assert L.dfm_fpn_missing_params(f.h) == 2
        outs = [torch.zeros(n * 64 * a * b, device='cuda') for a, b in sizes]
        assert f.forward(xs, outs) == 3                               # DFM_ERR_STATE
        assert f.debug('merged0', n * 64 * sizes[0][0] * sizes[0][1]) == 3
        v = f.host['lateral_convs.3.conv.weight']
        assert f.set('lateral_convs.3.conv.weight', v, v.numel() - 1) == 1   # DFM_ERR_INVALID
        assert f.set('fpn_convs.2.conv.bias', f.host['fpn_convs.2.conv.bias'], 63) == 1
        assert f.set('fpn_convs.9.conv.bias', f.host['fpn_convs.2.conv.bias']) == 1
        for k in skip:
            assert f.set(k, f.host[k]) == 0
        assert L.dfm_fpn_missing_params(f.h) == 0
        assert f.forward(xs, outs) == 0
        capi.sync_check()
        assert f.debug('merged0', n * 64 * sizes[0][0] * sizes[0][1]) == 0
        assert f.debug('fpn3', n * 64 * sizes[3][0] * sizes[3][1]) == 0
        assert f.debug('fpn3', 7) == 1
        assert f.debug('bogus', 7) == 1
        capi.sync_check()
    finally:
        f.close()
    # conv_impl='tc' with out_channels without a tensor-core kernel fails at create
    tc = _cuda_fpn(make_params(63, 32), 'tc', out_channels=32)
    with torch.no_grad(), pytest.raises(RuntimeError, match='no tensor-core kernel'):
        tc(xs)


@pytest.mark.gpu
def test_auto_falls_back_without_a_tensor_core_kernel():
    """out_channels = 32 has no tensor-core kernel: 'auto' runs the fp32 CUDA-core path (no
    tensor-core launch) and matches fp64 to fp32 rounding."""
    h, w, n = CASES['B']
    p = make_params(71, 32)
    xs = make_inputs(72, h, w, n, device='cuda')
    m = _cuda_fpn(p, out_channels=32)
    with torch.no_grad():
        m(xs)
        capi.sync_check()
        _, tc0 = capi.launch_counters()
        outs = m(xs)
        capi.sync_check()
        _, tc1 = capi.launch_counters()
        ref = fpn_forward({k: v.cuda().double() for k, v in p.items()}, [x.double() for x in xs])
    assert tc1 == tc0
    for got, r in zip(outs, ref):
        assert rel_err(got, r) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize('t,agg,neck', [(1, 'mean', 'imvoxel'), (2, 'concat', 'dfm')])
def test_waymo_fpn_to_box_regressions_end_to_end(t, agg, neck):
    """All-CUDA MultiViewDfM from the 2-D backbone's features (detectors/multiview_dfm.py:
    91-110, 119-268, 321-326): FPN -> lifting -> neck_3d -> Anchor3DHead against the all-oracle
    chain (fp64 FPN restatement, then the oracle lifting, neck and head), on the grid of
    test_waymo_box_regressions_end_to_end, for two samples with different metas."""
    from oracle import dfm_oracle as O
    from tests.test_anchor3d_head import _cuda_head, anchor3d_head_forward, load_fixture
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
    p = make_params(81)
    fpn = _cuda_fpn(p)
    p64 = {k: v.cuda().double() for k, v in p.items()}

    class Host(modules.MultiViewDfMFeatureTransformation):
        pass
    host = Host()
    host.n_voxels, host.voxel_range = n_voxels, vrange
    host.temporal_aggregate, host.valid_sample, host.neck_3d = agg, True, mod
    pyramids, metas = [], []
    for b in range(2):
        _, m = syn.make_waymo_sample(70 + b, t, nv, feat_hw=(40, 64), input_hw=(160, 256),
                                     flip=bool(b), scale=1.0 + 0.02 * b, crop=(1.0 * b, 2.0 * b))
        k = np.array([[120., 0, 128, 0], [0, 120., 80, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        full = syn.waymo_lidar2img(t, nv)
        kfull = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        m['ori_lidar2img'] = np.array([k @ np.linalg.inv(kfull) @ x for x in full])
        pyramids.append(make_inputs(90 + b, 160, 256, t * nv, device='cuda'))
        metas.append(m)
    with torch.no_grad():
        feats = [fpn(xs)[0] for xs in pyramids]                     # extract_feat, :91-110
        assert tuple(feats[0].shape) == (t * nv, 64, 40, 64)
        bev = host.feature_transformation(torch.stack(feats), metas, nv, t)[0]
        cls, box, dirc = head([bev])
    capi.sync_check()
    xs_, ys_, zs_ = modules.aligned_voxel_centers(n_voxels, vrange)
    zz, yy, xx = torch.meshgrid(zs_, ys_, xs_, indexing='ij')
    pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
    for b in range(2):
        m = metas[b]
        l2i = [torch.tensor(x, dtype=torch.float32) for x in m['ori_lidar2img']]
        with torch.no_grad():
            rfeat = fpn_forward(p64, [x.double() for x in pyramids[b]])[0].float().cpu()
            vol = O.multiview_lift(rfeat, pts, n_voxels, l2i, nv, t,
                                   pts.new_tensor(m['scale_factor'][:2]),
                                   pts.new_tensor(m['img_crop_offset']), m['flip'],
                                   m['input_shape'], m['img_shape'], agg)[None]
            rbev = (O.dfm_neck_forward(sd, vol, 64) if neck == 'dfm'
                    else O.imvoxel_neck_forward(sd, vol))[0]
            rcls, rbox, rdir = anchor3d_head_forward(hp, rbev)
        for got, ref, key in ((cls[0][b], rcls[0], 'cls_score'), (box[0][b], rbox[0], 'bbox_pred'),
                              (dirc[0][b], rdir[0], 'dir_cls_preds')):
            e = rel_err(got, ref)
            print('waymo fpn end to end', neck, b, key, e, 'worst element / tol',
                  assert_close(got, ref, key))
            assert e < 1e-3, (key, e)
