"""ResNet-101 with DCNv2 in layer3 / layer4 (mmdet's ``ResNet``, both MultiViewDfM Waymo configs'
``backbone``) on CUDA: fixture parity against an independent implementation (torchvision's
resnet101 with ``torchvision.ops.deform_conv2d``, tests/golden/make_resnet101_golden.py),
state_dict / registry / checkpoint plumbing, unsupported options, per-layer fp64 checks at the
shipped 832 x 1248 input, and the backbone feeding the FPN, lifting, 3-D neck and box head.

``resnet101_forward`` below is the fp32 / fp64 restatement of mmdet's forward (with
``deform_conv``, a gather-based modulated deformable conv) that the fixture checks; the GPU
tests compare against it.
"""
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import layer_check as LC
from tests.layer_check import SEPARATION, layer_bound
from tests.util import GOLDEN, assert_close

# must match tests/golden/make_resnet101_golden.py
CASES = {'small': (81, 2, 64, 96), 'odd': (82, 1, 70, 134)}
EDGE_CASES = ('odd',)
N_SAMPLE = 4096
STAGE_BLOCKS = (3, 4, 23, 3)
DCN = dict(type='DCNv2', deform_groups=1, fallback_on_stride=False)
FLOOR_C = 8.0
EW_TOL = 1e-5
REFERENCE_IO = json.load(open(os.path.join(GOLDEN, 'reference_io.json')))
WAYMO_CONFIGS = [k for k in REFERENCE_IO['configs'] if k.startswith('multiview-dfm_r101_dcn')]
BACKBONE_CFG = dict(REFERENCE_IO['configs'][WAYMO_CONFIGS[0]]['backbone'])
BACKBONE_CFG.pop('type')
HEADER = os.path.join(os.path.dirname(GOLDEN), '..', 'include', 'dfm_b200.h')


def blocks():
    """(name, stage, block index, stride, dcn) of the 33 Bottlenecks in forward order."""
    return [(f'layer{s + 1}.{j}', s, j, 2 if (j == 0 and s > 0) else 1, s >= 2)
            for s, n in enumerate(STAGE_BLOCKS) for j in range(n)]


# ---------------------------------------------------------------------------------------------
# fp32 / fp64 restatement of mmdet's ResNet forward with DCNv2
# ---------------------------------------------------------------------------------------------
def _bn(x, p, prefix):
    """Eval BatchNorm2d."""
    return F.batch_norm(x, p[prefix + '.running_mean'], p[prefix + '.running_var'],
                        p[prefix + '.weight'], p[prefix + '.bias'], False, 0.0, 1e-5)


def deform_columns(x, offset, mask, stride):
    """The [B, C, 9, Ho, Wo] samples of a modulated deformable 3x3 conv (pad 1): tap k = 3 ky +
    kx of output (y, x) reads x bilinearly at (y s - 1 + ky + offset[2k], x s - 1 + kx +
    offset[2k + 1]), each of the four corners outside the map counting as 0, times mask[k]."""
    b, c, h, w = x.shape
    ho, wo = offset.shape[2:]
    ys = (torch.arange(ho, device=x.device) * stride - 1).to(x.dtype)[:, None]
    xs = (torch.arange(wo, device=x.device) * stride - 1).to(x.dtype)[None, :]
    flat = x.reshape(b, c, h * w)
    cols = []
    for k in range(9):
        py = ys + k // 3 + offset[:, 2 * k]
        px = xs + k % 3 + offset[:, 2 * k + 1]
        y0, x0 = torch.floor(py), torch.floor(px)
        ly, lx = py - y0, px - x0
        val = 0
        for dy, dx, wt in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx),
                           (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
            yy, xx = y0 + dy, x0 + dx
            ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
            idx = (yy.clamp(0, h - 1) * w + xx.clamp(0, w - 1)).long().reshape(b, 1, -1)
            v = torch.gather(flat, 2, idx.expand(b, c, -1)).view(b, c, ho, wo)
            val = val + v * (wt * ok)[:, None]
        cols.append(val * mask[:, k:k + 1])
    return torch.stack(cols, 2)


def deform_conv(x, offset, mask, w, stride):
    cols = deform_columns(x, offset, mask, stride)
    return torch.einsum('bckhw,ock->bohw', cols, w.reshape(w.shape[0], w.shape[1], 9))


def resnet101_forward(p, img, with_intermediates=False):
    """mmdet ResNet.forward (depth 101, style 'pytorch', max-pool stem) with
    Bottleneck.forward: relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1(x)))))))) + identity), the
    stride in conv2, and in layer3 / layer4 conv2 = ModulatedDeformConv2dPack (o = conv_offset(x);
    offsets o[:, :18], masks sigmoid(o[:, 18:])).  Returns the 4 stage outputs (and a dict of
    intermediates)."""
    x = F.relu(_bn(F.conv2d(img, p['conv1.weight'], None, 2, 3), p, 'bn1'))
    mid = {'stem_act': x}
    x = F.max_pool2d(x, 3, 2, 1)
    mid['pool'] = x
    outs = []
    for name, s, j, stride, dcn in blocks():
        mid[name + '.in'] = x
        a1 = F.relu(_bn(F.conv2d(x, p[name + '.conv1.weight']), p, name + '.bn1'))
        mid[name + '.a1'] = a1
        if dcn:
            o = F.conv2d(a1, p[name + '.conv2.conv_offset.weight'],
                         p[name + '.conv2.conv_offset.bias'], stride, 1)
            mid[name + '.om'] = o
            a2 = deform_conv(a1, o[:, :18], torch.sigmoid(o[:, 18:]), p[name + '.conv2.weight'],
                             stride)
        else:
            a2 = F.conv2d(a1, p[name + '.conv2.weight'], None, stride, 1)
        a2 = F.relu(_bn(a2, p, name + '.bn2'))
        mid[name + '.a2'] = a2
        y = _bn(F.conv2d(a2, p[name + '.conv3.weight']), p, name + '.bn3')
        if j == 0:
            x = _bn(F.conv2d(x, p[name + '.downsample.0.weight'], None, stride), p,
                    name + '.downsample.1')
        x = F.relu(y + x)
        mid[name] = x
        if j == STAGE_BLOCKS[s] - 1:
            outs.append(x)
    return (tuple(outs), mid) if with_intermediates else tuple(outs)


def load_case(name):
    from depth_from_motion_b200 import synthetic as syn
    seed, b, h, w = CASES[name]
    img, sd = syn.make_resnet101_case(seed, h, w, b)
    gold = dict(np.load(os.path.join(GOLDEN, 'resnet101_dcn.npz')))
    return img, sd, gold, (seed, b, h, w)


def check_against_fixture(name, outs):
    img, sd, gold, (seed, b, h, w) = load_case(name)
    worst = {}
    for lvl, o in enumerate(outs):
        o = o.detach().cpu()
        n = o[0].numel()
        idx = torch.from_numpy(np.random.RandomState(seed + 100 * (lvl + 1)).randint(0, n, N_SAMPLE))
        got = torch.stack([o[i].reshape(-1)[idx] for i in range(b)])
        worst[f'out{lvl}'] = assert_close(got, gold[f'{name}_out{lvl}_sample'], f'{name} out{lvl}')
        if name in EDGE_CASES:
            th, tw = o.shape[2:]
            worst[f'out{lvl}_rows'] = assert_close(o[:, :, [0, th - 1], :],
                                                   gold[f'{name}_out{lvl}_rows'], 'rows')
            worst[f'out{lvl}_cols'] = assert_close(o[:, :, :, [0, tw - 1]],
                                                   gold[f'{name}_out{lvl}_cols'], 'cols')
    return worst


def fp64_params(sd, dev='cpu'):
    return {k: v.to(dev, torch.float64) for k, v in sd.items() if v.is_floating_point()}


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(CASES))
def test_restatement_reproduces_fixture(name):
    img, sd, gold, _ = load_case(name)
    np.testing.assert_allclose([img.double().sum().item(), img.double().abs().sum().item()],
                               gold[f'{name}_img_sums'], rtol=1e-9)
    np.testing.assert_allclose(sum(v.double().abs().sum().item() for v in sd.values()),
                               gold[f'{name}_w_abs'], rtol=1e-9)
    with torch.no_grad():
        print(name, 'fp32', check_against_fixture(name, resnet101_forward(sd, img)))
        outs, mid = resnet101_forward(fp64_params(sd), img.double(), with_intermediates=True)
        print(name, 'fp64', check_against_fixture(name, outs))
    # the synthetic conv_offset moves samples by several pixels and off the map
    o = mid['layer3.0.om'][:, :18].abs()
    assert float(o.max()) > 3.0 and float((o > 1.0).double().mean()) > 0.2, float(o.max())


def test_deform_restatement_matches_torchvision():
    tv = pytest.importorskip('torchvision.ops')
    g = torch.Generator().manual_seed(5)
    for stride, (h, w) in ((1, (9, 13)), (2, (11, 8))):
        x = torch.randn(2, 16, h, w, generator=g, dtype=torch.float64)
        ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
        off = 3.0 * torch.randn(2, 18, ho, wo, generator=g, dtype=torch.float64)
        off[:, :, 0, 0] = torch.round(off[:, :, 0, 0])          # integer positions too
        mask = torch.rand(2, 9, ho, wo, generator=g, dtype=torch.float64)
        wt = torch.randn(8, 16, 3, 3, generator=g, dtype=torch.float64)
        ref = tv.deform_conv2d(x, off, wt, None, stride=stride, padding=1, mask=mask)
        got = deform_conv(x, off, mask, wt, stride)
        assert float((got - ref).abs().max()) < 1e-12 * float(ref.abs().max()), stride


@pytest.mark.parametrize('axis', ['dy', 'dx'])
def test_integer_offset_identity(axis):
    """dy = 1 (or dx = 1) on every tap with mask 1 reads the zero-padded input one row (column)
    further on: F.conv2d(F.pad(x, (1, 2, 1, 2)), w) shifted by one output row (column).  Pins
    channel 2k = dy, 2k + 1 = dx without any library."""
    g = torch.Generator().manual_seed(6)
    h, w = 7, 10
    x = torch.randn(1, 5, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(4, 5, 3, 3, generator=g, dtype=torch.float64)
    off = torch.zeros(1, 18, h, w, dtype=torch.float64)
    off[:, 0 if axis == 'dy' else 1::2] = 1.0
    got = deform_conv(x, off, torch.ones(1, 9, h, w, dtype=torch.float64), wt, 1)
    full = F.conv2d(F.pad(x, (1, 2, 1, 2)), wt)
    ref = full[..., 1:h + 1, 0:w] if axis == 'dy' else full[..., 0:h, 1:w + 1]
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)


def test_mirror_state_dict_matches_reference():
    from depth_from_motion_b200 import modules
    gold = dict(np.load(os.path.join(GOLDEN, 'resnet101_dcn.npz')))
    sd = modules.ResNet(**BACKBONE_CFG).state_dict()
    assert list(sd) == list(gold['state_keys'])
    assert [','.join(str(n) for n in v.shape) for v in sd.values()] == list(gold['state_shapes'])
    assert len(sd) == 676 and sum(v.numel() for v in sd.values()) == 44410342
    _, ref_sd, _, _ = load_case('small')
    modules.ResNet(**BACKBONE_CFG).load_state_dict(ref_sd, strict=True)


@pytest.mark.parametrize('cfg_name', WAYMO_CONFIGS)
def test_waymo_configs_build_resnet(cfg_name):
    from depth_from_motion_b200 import modules, registry
    cfg = REFERENCE_IO['configs'][cfg_name]['backbone']
    m = registry.build_backbone(dict(cfg))
    assert type(m) is modules.ResNet and m.depth == 101
    assert m.stage_with_dcn == (False, False, True, True)
    from oracle.ref_loader import REFERENCE_ROOT
    ref = os.path.join(REFERENCE_ROOT, 'configs', 'dfm', cfg_name)
    if os.path.isfile(ref):
        direct = registry.Config.fromfile(ref).model['backbone']
        assert type(registry.build_backbone(dict(direct))) is modules.ResNet


@pytest.mark.parametrize('change', [
    dict(depth=50), dict(depth=34), dict(dcn=None), dict(stage_with_dcn=(False, True, True, True)),
    dict(dcn=dict(type='DCN', deform_groups=1, fallback_on_stride=False)),
    dict(dcn=dict(type='DCNv2', deform_groups=2, fallback_on_stride=False)),
    dict(dcn=dict(type='DCNv2', deform_groups=1, fallback_on_stride=True)),
    dict(style='caffe'), dict(strides=(1, 2, 2, 1)), dict(dilations=(1, 1, 1, 2)),
    dict(out_indices=(1, 2, 3)), dict(deep_stem=True), dict(avg_down=True),
    dict(plugins=[dict(cfg=dict(type='ContextBlock'), position='after_conv3')]),
    dict(norm_cfg=dict(type='GN', num_groups=32)), dict(conv_cfg=dict(type='ConvWS')),
    dict(num_stages=3)])
def test_unsupported_options_raise(change):
    from depth_from_motion_b200 import modules
    with pytest.raises(NotImplementedError):
        modules.ResNet(**dict(BACKBONE_CFG, **change))


def test_ignored_options_accepted():
    from depth_from_motion_b200 import modules
    for change in (dict(frozen_stages=-1), dict(norm_eval=False), dict(init_cfg=None),
                   dict(pretrained='x.pth', init_cfg=None), dict(with_cp=True),
                   dict(zero_init_residual=False), dict(norm_cfg=dict(type='SyncBN'))):
        modules.ResNet(**dict(BACKBONE_CFG, **change))


def test_input_validation_before_any_launch():
    from depth_from_motion_b200 import modules
    m = modules.ResNet(**BACKBONE_CFG).eval()
    for bad in (torch.zeros(3, 32, 32), torch.zeros(1, 4, 32, 32), torch.zeros(1, 1, 32, 32),
                torch.zeros(1, 3, 0, 32), torch.zeros(1, 3, 32, 0)):
        with pytest.raises(ValueError):
            m(bad)
    assert m._handle is None
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        m(torch.zeros(1, 3, 32, 32))
    m.train()
    with pytest.raises(RuntimeError):
        m._forward_only(torch.zeros(1, requires_grad=True))


def test_load_hot_path_loads_img_backbone():
    from depth_from_motion_b200 import checkpoint, modules
    _, sd, _, _ = load_case('small')
    m = modules.ResNet(**BACKBONE_CFG)
    full = {'backbone.' + k: v for k, v in sd.items()}
    full['neck.lateral_convs.0.conv.weight'] = torch.zeros(1)
    full['bbox_head_3d.conv_cls.weight'] = torch.zeros(1)
    res = checkpoint.load_hot_path({'state_dict': full}, img_backbone=m)
    assert not res['backbone'].missing_keys and not res['backbone'].unexpected_keys
    k = 'layer3.7.conv2.conv_offset.weight'
    assert torch.equal(m.state_dict()[k], sd[k])
    assert torch.equal(m.state_dict()['layer4.2.bn3.running_var'], sd['layer4.2.bn3.running_var'])
    with pytest.raises(KeyError, match='"backbone."'):
        checkpoint.load_hot_path({'state_dict': {'neck.x': torch.zeros(1)}},
                                 img_backbone=modules.ResNet(**BACKBONE_CFG))


def test_descriptor_matches_header():
    from depth_from_motion_b200 import capi
    src = open(HEADER).read()
    body = re.search(r'typedef struct dfm_resnet101_desc \{(.*?)\} dfm_resnet101_desc_t;',
                     src, re.S).group(1)
    fields = re.findall(r'int (\w+);', body)
    assert fields == [f for f, _ in capi.ResNet101Desc._fields_]
    for fn in ('create', 'destroy', 'set_param', 'missing_params', 'forward', 'debug_tensor'):
        assert f'dfm_resnet101_{fn}' in capi.SYMBOLS
        assert f'dfm_resnet101_{fn}(' in src


def test_output_sizes_follow_pytorch():
    from depth_from_motion_b200 import modules
    for h, w in ((832, 1248), (70, 134), (71, 1), (1, 3), (33, 65)):
        x = torch.zeros(1, 1, h, w)
        sizes = [F.conv2d(x, torch.zeros(1, 1, 7, 7), None, 2, 3)]
        sizes.append(F.max_pool2d(sizes[-1], 3, 2, 1))
        for _ in range(3):
            a = F.conv2d(sizes[-1], torch.zeros(1, 1, 3, 3), None, 2, 1)
            assert a.shape == F.conv2d(sizes[-1], torch.zeros(1, 1, 1, 1), None, 2).shape
            sizes.append(a)
        assert modules.ResNet.output_sizes(h, w) == [tuple(s.shape[2:]) for s in sizes]


# --- per-layer error model: bf16-split emulation, for plain and deformable convs ---
def conv64(x, w, stride=1, om=None):
    """A conv of the backbone in fp64: 1x1 (pad 0), 3x3 (pad 1) or, with om = [B, 27 (+), H, W]
    offsets | sigmoid masks, the modulated deformable 3x3."""
    if om is not None:
        return deform_conv(x, om[:, :18], om[:, 18:27], w, stride)
    return F.conv2d(x, w, None, stride, w.shape[-1] // 2)


def emulated(x, w, stride=1, om=None):
    """The 3-term split and its two 2-term variants, in fp64.  For a deformable conv the split
    operand is the blended, masked sample (what the loaders split), not the input map."""
    if om is not None:
        cols = deform_columns(x, om[:, :18], om[:, 18:27], stride)
        ch, cl = LC.split16(cols)
        wh, wl = LC.split16(w.reshape(w.shape[0], w.shape[1], 9))

        def mm(a, b):
            return torch.einsum('bckhw,ock->bohw', a, b)
        a, b, c = mm(ch, wh), mm(cl, wh), mm(ch, wl)
    else:
        xh, xl = LC.split16(x)
        wh, wl = LC.split16(w)
        a, b, c = conv64(xh, wh, stride), conv64(xl, wh, stride), conv64(xh, wl, stride)
    return a + b + c, a + c, a + b


def layer_classes(sd, img):
    """(label, input, weight, stride, om) of one layer of each new class, fp64: 1x1 (K = 64 ..
    2048, stride 1 and 2), the plain stride-2 3x3, conv_offset, the deformable conv (stride 1, 2)."""
    p = fp64_params(sd)
    with torch.no_grad():
        _, mid = resnet101_forward(p, img.double(), with_intermediates=True)
    om = {n: torch.cat([mid[n + '.om'][:, :18], torch.sigmoid(mid[n + '.om'][:, 18:])], 1)
          for n in ('layer3.0', 'layer3.1', 'layer4.0')}
    return [('layer1.0.conv1', mid['layer1.0.in'], p['layer1.0.conv1.weight'], 1, None),
            ('layer3.2.conv3', mid['layer3.2.a2'], p['layer3.2.conv3.weight'], 1, None),
            ('layer4.0.downsample', mid['layer4.0.in'], p['layer4.0.downsample.0.weight'], 2, None),
            ('layer4.1.conv1', mid['layer4.1.in'], p['layer4.1.conv1.weight'], 1, None),
            ('layer2.0.conv2', mid['layer2.0.a1'], p['layer2.0.conv2.weight'], 2, None),
            ('layer3.1.conv_offset', mid['layer3.1.a1'], p['layer3.1.conv2.conv_offset.weight'], 1,
             None),
            ('layer3.0.conv2', mid['layer3.0.a1'], p['layer3.0.conv2.weight'], 2, om['layer3.0']),
            ('layer3.1.conv2', mid['layer3.1.a1'], p['layer3.1.conv2.weight'], 1, om['layer3.1']),
            ('layer4.0.conv2', mid['layer4.0.a1'], p['layer4.0.conv2.weight'], 2, om['layer4.0'])]


def test_bound_separates_lost_term_cpu():
    img, sd, _, _ = load_case('odd')
    for label, x, w, stride, om in layer_classes(sd, img):
        ref = conv64(x, w, stride, om)
        e3, e2 = LC.norm_errors(emulated(x, w, stride, om), ref)
        k = w.shape[1] * w.shape[2] * w.shape[3]
        bound = layer_bound(e3, k, FLOOR_C)
        print(f'{label}: K {k} e3 {e3:.2e} e2 {e2:.2e} bound {bound:.2e} e2/bound {e2 / bound:.1f}')
        assert SEPARATION * bound <= e2, (label, bound, e2)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
N_TC = 33 * 3 + 4 + 26        # conv1 / conv2 / conv3 of every block, 4 downsamples, 26 conv_offset


def make_backbone(sd, impl='auto'):
    from depth_from_motion_b200 import modules
    m = modules.ResNet(**BACKBONE_CFG, conv_impl=impl)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _tc_count(fn):
    from depth_from_motion_b200 import capi
    _, t0 = capi.launch_counters()
    out = fn()
    capi.sync_check()
    _, t1 = capi.launch_counters()
    return out, t1 - t0


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['simt', 'auto'])
@pytest.mark.parametrize('name', list(CASES))
def test_fixture_parity(name, impl):
    img, sd, _, _ = load_case(name)
    m = make_backbone(sd, impl)
    with torch.no_grad():
        m(img.cuda())
        outs, tc = _tc_count(lambda: m(img.cuda()))
    # every conv but the stem runs on tensor cores under auto
    assert tc == (N_TC if impl == 'auto' else 0), tc
    print(name, impl, check_against_fixture(name, outs))


WHOLE_CASES = {'waymo5': (91, 5, 832, 1248, ('auto',)), 'odd': (82, 1, 70, 134, ('auto', 'simt')),
               'small': (81, 2, 64, 96, ('auto', 'simt'))}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(WHOLE_CASES))
def test_whole_module_vs_fp64(case):
    from depth_from_motion_b200 import synthetic as syn
    seed, b, h, w, impls = WHOLE_CASES[case]
    img, sd = syn.make_resnet101_case(seed, h, w, b)
    with torch.no_grad():
        ref = resnet101_forward(fp64_params(sd, 'cuda'), img.cuda().double())
        for impl in impls:
            outs = make_backbone(sd, impl)(img.cuda())
            for lvl, (o, r) in enumerate(zip(outs, ref)):
                assert o.shape == r.shape
                print(case, impl, lvl, assert_close(o, r, f'{case} {impl} out{lvl}'))
    torch.cuda.empty_cache()


def _shell(n, tile):
    """Output indices at either border and, for a pixel-row tile, all of them (1-D tiles of
    128 flattened pixels cut rows anywhere: the shell is the first / last row and column)."""
    i = torch.arange(n)
    return (i < 1) | (i >= n - 1)


class LayerChecker:
    """One row per conv: the GPU's raw output against fp64 from the GPU's own input (and, for a
    deformable conv, the GPU's own offsets and masks), the bound max(6 e3, 8 sqrt(K) 2^-24)
    (the accumulation floor alone for CUDA-core layers), that bound >= 3x below the lost-term
    error e2, and the element-wise form on the border rows / columns and the tile seams."""

    def __init__(self):
        self.rows, self.failures, self.checked = [], [], set()

    def conv(self, label, got, x, w, cls, tc, stride=1, om=None):
        ref = conv64(x, w, stride, om)
        ys = emulated(x, w, stride, om)
        k = w.shape[1] * w.shape[2] * w.shape[3]
        assert got.shape == ref.shape, (label, got.shape, ref.shape)
        e = float((got - ref).abs().max() / ref.abs().max())
        e3, e2 = LC.norm_errors(ys, ref)
        bound = layer_bound(e3, k, FLOOR_C) if tc else LC.acc_floor(k, FLOOR_C)
        row = dict(layer=label, cls=cls, err=e, e3=e3, e2=e2, bound=bound)
        if e > bound:
            self.failures.append((label, e, bound))
        if tc and SEPARATION * bound > e2:
            self.failures.append((label, 'separation', bound, e2))
        if tc:
            if om is not None:
                sc = deform_conv(x.abs(), om[:, :18], om[:, 18:27], w.abs(), stride)
            else:
                sc = conv64(x.abs(), w.abs(), stride)
            b, _, hh, ww = got.shape
            # borders, plus every pixel whose flattened index sits at a 128-row tile seam
            m = _shell(hh, 0)[:, None] | _shell(ww, 0)[None, :]
            m = m[None].expand(b, hh, ww).clone()
            flat = torch.arange(b * hh * ww).view(b, hh, ww)
            m |= (flat % 128 == 0) | (flat % 128 == 127)
            m = m.to(got.device)
            sel = [t.movedim(1, -1)[m] for t in (got, ref) + tuple(ys) + (sc,)]
            eg, _, el2, elb = LC.elementwise_errors(*sel, k, FLOOR_C)
            row.update(shell=eg, shell_bound=elb, shell_e2=el2)
            if eg > elb:
                self.failures.append((label, 'shell element', eg, elb))
            if SEPARATION * elb > el2:
                self.failures.append((label, 'shell separation', elb, el2))
        self.rows.append(row)
        self.checked.add(cls)

    def elementwise(self, label, got, ref, tol=EW_TOL):
        e = float((got - ref).abs().max() / ref.abs().max())
        self.rows.append(dict(layer=label, cls='elementwise', err=e, bound=tol))
        if e > tol:
            self.failures.append((label, e, tol))

    def report(self, case):
        nan = float('nan')
        for r in self.rows:
            print(f"{case} | {r['layer']} | {r['cls']} | {r['err']:.2e} | {r['bound']:.2e} | "
                  f"{r.get('e3', nan):.2e} | {r.get('e2', nan):.2e} || {r.get('shell', nan):.2e} | "
                  f"{r.get('shell_bound', nan):.2e} | {r.get('shell_e2', nan):.2e}")


CHECK_BLOCKS = ('layer1.0', 'layer1.2', 'layer2.0', 'layer2.1', 'layer3.0', 'layer3.11',
                'layer3.22', 'layer4.0', 'layer4.2')


def run_layers(seed, b, h, w, impl='auto', names=CHECK_BLOCKS):
    from depth_from_motion_b200 import synthetic as syn
    from tests.test_stage_layers import profiled
    img, sd = syn.make_resnet101_case(seed, h, w, b)
    m = make_backbone(sd, impl)
    img = img.cuda()
    _, report = profiled(lambda: m(img))
    p = fp64_params(sd, 'cuda')
    sizes = m.output_sizes(h, w)
    ck = LayerChecker()
    tc_on = impl != 'simt'

    def dbg(name, hw, c):
        return m.debug_tensor(name, (b,) + hw + (c,)).permute(0, 3, 1, 2).double()

    def folded(x, prefix, relu):
        s = p[prefix + '.weight'] / torch.sqrt(p[prefix + '.running_var'] + 1e-5)
        sh = (p[prefix + '.bias'] - p[prefix + '.running_mean'] * s).float().double()
        y = x * s.float().double()[:, None, None] + sh[:, None, None]
        return F.relu(y) if relu else y

    def cls(kind, cin, cout, k, s, tag=''):
        return f'{kind}<{cin}->{cout},k{k},s{s}{tag}'

    g = 'rn101_gather_tc' if tc_on else 'rn101_conv_simt'
    stem = dbg('stem', sizes[0], 64)
    ck.conv('stem', stem, img.double(), p['conv1.weight'], 'resnet_stem', False, 2)
    # bn1 + ReLU + max-pool is exact in fp32 up to the folded affine's rounding
    pool = dbg('pool', sizes[1], 64)
    ck.elementwise('pool', pool, F.max_pool2d(folded(stem, 'bn1', True), 3, 2, 1))
    order = [n for n, *_ in blocks()]
    for name, s, j, stride, dcn in blocks():
        if name not in names:
            continue
        planes = 64 << s
        hin = sizes[s] if (j == 0 and s > 0) else sizes[s + 1]
        hout = sizes[s + 1]
        i = order.index(name)
        x = pool if i == 0 else dbg(order[i - 1], hin, (planes * 2) if j == 0 else planes * 4)
        cin = x.shape[1]
        r1 = dbg(name + '.conv1', hin, planes)
        ck.conv(name + '.conv1', r1, x, p[name + '.conv1.weight'], cls(g, cin, planes, 1, 1),
                tc_on)
        a1 = folded(r1, name + '.bn1', True)
        om = None
        if dcn:
            ro = dbg(name + '.conv2.conv_offset', hout, 32)[:, :27]
            ck.conv(name + '.conv_offset', ro - p[name + '.conv2.conv_offset.bias'][:, None, None],
                    a1, p[name + '.conv2.conv_offset.weight'], cls(g, planes, 27, 3, stride, ',off'),
                    tc_on, stride)
            om = dbg(name + '.conv2.offset_mask', hout, 32)
            ck.elementwise(name + '.offset_mask', om[:, :27],
                           torch.cat([ro[:, :18], torch.sigmoid(ro[:, 18:])], 1), tol=1e-6)
        r2 = dbg(name + '.conv2', hout, planes)
        if dcn:
            c2 = cls(g, planes, planes, 3, stride, ',dcn')
        elif stride == 1 and tc_on:
            c2 = f'resnet_conv_tc<{planes}->{planes},k3,s1,d1'
        else:
            c2 = cls(g, planes, planes, 3, stride)
        ck.conv(name + '.conv2', r2, a1, p[name + '.conv2.weight'], c2, tc_on, stride, om)
        a2 = folded(r2, name + '.bn2', True)
        identity = x
        if j == 0:
            rd = dbg(name + '.downsample', hout, 4 * planes)
            ck.conv(name + '.downsample', rd, x, p[name + '.downsample.0.weight'],
                    cls(g, cin, 4 * planes, 1, stride), tc_on, stride)
            identity = folded(rd, name + '.downsample.1', False)
        r3 = dbg(name + '.conv3', hout, 4 * planes)
        ck.conv(name + '.conv3', r3, a2, p[name + '.conv3.weight'], cls(g, planes, 4 * planes, 1, 1),
                tc_on)
        out = dbg(name, hout, 4 * planes)
        ck.elementwise(name, out, F.relu(folded(r3, name + '.bn3', False) + identity))
        torch.cuda.empty_cache()
    tc_kinds = ('rn101_gather_tc<', 'resnet_conv_tc<')
    launched = {k.split('>@')[0] for k in report if k.startswith(tc_kinds)}
    if launched - ck.checked:
        ck.failures.append(('tensor-core classes launched but not compared',
                            sorted(launched - ck.checked)))
    ck.report(f'resnet101 {b}x{h}x{w} {impl}')
    print('CLASSES', ' '.join(sorted(report)))
    return ck, launched


@pytest.mark.gpu
def test_layers_vs_fp64_waymo_shape():
    """Two 832 x 1248 views in one call: tiles straddle the images' seam."""
    ck, launched = run_layers(92, 2, 832, 1248)
    assert not ck.failures, ck.failures
    assert any(',dcn' in c for c in launched) and any(',off' in c for c in launched)


@pytest.mark.gpu
def test_layers_vs_fp64_simt():
    ck, launched = run_layers(93, 1, 70, 134, impl='simt')
    assert not launched
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_c_api_errors_and_repeatability():
    from depth_from_motion_b200 import capi
    L = capi.lib()
    img, sd, _, (_, b, h, w) = load_case('odd')
    for bad in ((0, 20, 1, 0), (20, 20, 0, 0), (20, 20, 1, 7), (100000, 100000, 1, 0)):
        hd = ctypes.c_void_p()
        assert L.dfm_resnet101_create(ctypes.byref(capi.ResNet101Desc(*bad)),
                                      ctypes.byref(hd)) == 1, bad
    hd = ctypes.c_void_p()
    assert L.dfm_resnet101_create(ctypes.byref(capi.ResNet101Desc(h, w, b, capi.DFM_CONV_TC)),
                                  ctypes.byref(hd)) == 0
    keys = [k for k in sd if not k.endswith('num_batches_tracked')]
    assert L.dfm_resnet101_missing_params(hd) == len(keys) == 572

    def put(k, v, n=None):
        v = v.float().contiguous()
        return L.dfm_resnet101_set_param(hd, k.encode(), ctypes.c_void_p(v.data_ptr()),
                                         v.numel() if n is None else n)
    for k in keys[:-1]:
        assert put(k, sd[k]) == 0, k
    from depth_from_motion_b200 import modules
    sizes = modules.ResNet.output_sizes(h, w)
    outs = [torch.empty((b, 256 << l) + sizes[l + 1], device='cuda') for l in range(4)]
    arr = (ctypes.c_void_p * 4)(*[o.data_ptr() for o in outs])
    x = img.cuda().contiguous()
    assert L.dfm_resnet101_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 3
    assert put(keys[-1], sd[keys[-1]], 7) == 1
    assert put('layer5.0.conv1.weight', sd[keys[-1]]) == 1
    assert put('layer1.0.conv2.conv_offset.weight', sd['layer3.0.conv2.conv_offset.weight']) == 1
    assert put('layer3.0.conv2.conv_offset.bias', sd['layer3.0.conv2.conv_offset.bias'], 32) == 1
    assert put(keys[-1], sd[keys[-1]]) == 0
    buf = torch.empty(b * sizes[0][0] * sizes[0][1] * 64, device='cuda')
    assert L.dfm_resnet101_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                        buf.numel(), None) == 3
    _, t0 = capi.launch_counters()
    assert L.dfm_resnet101_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 0
    capi.sync_check()
    _, t1 = capi.launch_counters()
    assert t1 - t0 == N_TC
    first = [o.clone() for o in outs]
    assert L.dfm_resnet101_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 0
    capi.sync_check()
    assert all(torch.equal(a, o) for a, o in zip(first, outs))       # bitwise repeatable
    assert L.dfm_resnet101_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                        buf.numel(), None) == 0
    assert L.dfm_resnet101_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                        buf.numel() - 1, None) == 1
    assert L.dfm_resnet101_debug_tensor(hd, b'layer5.0', ctypes.c_void_p(buf.data_ptr()),
                                        buf.numel(), None) == 1
    L.dfm_resnet101_destroy(hd)
    # no overrun: each output is written exactly, the guard after it untouched
    m = make_backbone(sd)
    with torch.no_grad():
        ref = m(img.cuda())
        guard = [torch.full((o.numel() + 4096,), 7.0, device='cuda') for o in ref]
        arr = (ctypes.c_void_p * 4)(*[g.data_ptr() for g in guard])
        capi.check(L.dfm_resnet101_forward(m._handle, ctypes.c_void_p(x.data_ptr()), arr, None),
                   'forward')
        capi.sync_check()
        for g, o in zip(guard, ref):
            assert torch.equal(g[:o.numel()].view_as(o), o)
            assert bool((g[o.numel():] == 7.0).all())
        # a batch of two gives each image what a batch of one gives it
        two = m(torch.cat((img, img.flip(-1))).cuda())
        one = m(img.flip(-1).cuda())
    assert all(torch.equal(t[:1], f) for t, f in zip(two, first))
    assert all(torch.equal(t[1:], o) for t, o in zip(two, one))
    assert not math.isnan(float(two[3].sum()))


@pytest.mark.gpu
@pytest.mark.parametrize('t,agg,neck', [(1, 'mean', 'imvoxel'), (2, 'concat', 'dfm')])
def test_waymo_images_to_box_regressions_end_to_end(t, agg, neck):
    """All-CUDA MultiViewDfM from the normalised images: ResNet -> FPN -> lifting -> neck_3d ->
    Anchor3DHead against the all-oracle chain (fp64 ResNet and FPN restatements, then the oracle
    lifting, neck and head), on the grid of test_waymo_fpn_to_box_regressions_end_to_end."""
    from oracle import dfm_oracle as O
    from depth_from_motion_b200 import capi, modules
    from depth_from_motion_b200 import synthetic as syn
    from tests.test_anchor3d_head import _cuda_head, anchor3d_head_forward, load_fixture
    from tests.test_fpn import _cuda_fpn, fpn_forward, make_params
    from tests.util import rel_err
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
    _, bsd = syn.make_resnet101_case(94, 8, 8, 1)
    bb = make_backbone(bsd)
    b64 = fp64_params(bsd, 'cuda')

    class Host(modules.MultiViewDfMFeatureTransformation):
        pass
    host = Host()
    host.n_voxels, host.voxel_range = n_voxels, vrange
    host.temporal_aggregate, host.valid_sample, host.neck_3d = agg, True, mod
    imgs, metas = [], []
    for b in range(2):
        _, m = syn.make_waymo_sample(70 + b, t, nv, feat_hw=(40, 64), input_hw=(160, 256),
                                     flip=bool(b), scale=1.0 + 0.02 * b, crop=(1.0 * b, 2.0 * b))
        k = np.array([[120., 0, 128, 0], [0, 120., 80, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        full = syn.waymo_lidar2img(t, nv)
        kfull = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        m['ori_lidar2img'] = np.array([k @ np.linalg.inv(kfull) @ x for x in full])
        imgs.append(syn.make_resnet101_case(95 + b, 160, 256, t * nv)[0].cuda())
        metas.append(m)
    with torch.no_grad():
        feats = [fpn(list(bb(x)))[0] for x in imgs]                  # extract_feat
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
            rb = resnet101_forward(b64, imgs[b].double())
            rfeat = fpn_forward(p64, list(rb))[0].float().cpu()
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
            print('waymo images end to end', neck, b, key, e, 'worst element / tol',
                  assert_close(got, ref, key))
            assert e < 1e-3, (key, e)
