"""LIGAResNet-34 (backbones/liga_resnet.py, shipped KITTI config) on CUDA: fixture parity against
the reference module, state_dict / registry / checkpoint plumbing, unsupported options, per-layer
fp64 checks at the benchmarked 384 x 1248 input, and the backbone feeding SPPUNetNeck.

``liga_resnet_forward`` below is the fp32 / fp64 restatement of the reference forward that the
fixture (tests/golden/make_liga_resnet_golden.py) checks; the GPU tests compare against it.
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

# must match tests/golden/make_liga_resnet_golden.py
CASES = {'small': (51, 2, 64, 160), 'odd': (52, 1, 70, 134)}
EDGE_CASES = ('odd',)
N_SAMPLE = 4096
BACKBONE_CFG = dict(depth=34, num_stages=4, strides=(1, 2, 1, 1), dilations=(1, 1, 2, 4),
                    out_indices=(0, 1, 2, 3), style='pytorch', frozen_stages=-1,
                    norm_cfg=dict(type='SyncBN', requires_grad=True), norm_eval=False,
                    with_max_pool=False, block_with_final_relu=False,
                    num_channels_factor=(1, 2, 2, 2))
STAGES = ((3, 64, 1), (4, 128, 1), (6, 128, 2), (3, 128, 4))   # blocks, channels, dilation
TILE = (16, 8)          # resnet_conv_tc_kernel: 16 output rows x 8 output columns
FLOOR_C = 8.0
EW_TOL = 1e-5
REFERENCE_IO = json.load(open(os.path.join(GOLDEN, 'reference_io.json')))
HEADER = os.path.join(os.path.dirname(GOLDEN), '..', 'include', 'dfm_b200.h')


def blocks():
    """(name, stage index, block index, stride, dilation) of the 16 blocks in forward order."""
    out = []
    for s, (n, _, d) in enumerate(STAGES):
        for j in range(n):
            out.append((f'layer{s + 1}.{j}', s, j, 2 if (s == 1 and j == 0) else 1, d))
    return out


# ---------------------------------------------------------------------------------------------
# fp32 / fp64 restatement of the reference forward
# ---------------------------------------------------------------------------------------------
def _bn(x, p, prefix):
    """Eval BatchNorm2d / SyncBatchNorm."""
    return F.batch_norm(x, p[prefix + '.running_mean'], p[prefix + '.running_var'],
                        p[prefix + '.weight'], p[prefix + '.bias'], False, 0.0, 1e-5)


def liga_resnet_forward(p, img, with_intermediates=False):
    """LIGAResNet.forward (liga_resnet.py:467-483) with LigaBasicBlock.forward (:66-94) for the
    KITTI config: stem 7x7 / 2 + BN + ReLU, no max-pool; blocks bn2(conv2(relu(bn1(conv1(x)))))
    + identity without a final ReLU; conv1 of every block has the stage's dilation (padding =
    dilation), layer2.0 has stride 2 and a 1x1 / 2 downsample.  Returns the 4 stage outputs
    (and a dict of every block's input, conv1 input and output)."""
    x = F.relu(_bn(F.conv2d(img, p['conv1.weight'], None, 2, 3), p, 'bn1'))
    mid, outs = {'stem_act': x}, []
    for name, s, j, stride, d in blocks():
        mid[name + '.in'] = x
        a = F.conv2d(x, p[name + '.conv1.weight'], None, stride, d, d)
        a = F.relu(_bn(a, p, name + '.bn1'))
        mid[name + '.a1'] = a
        y = _bn(F.conv2d(a, p[name + '.conv2.weight'], None, 1, 1), p, name + '.bn2')
        if name + '.downsample.0.weight' in p:
            x = _bn(F.conv2d(x, p[name + '.downsample.0.weight'], None, stride), p,
                    name + '.downsample.1')
        x = y + x
        mid[name] = x
        if j == STAGES[s][0] - 1:
            outs.append(x)
    return (tuple(outs), mid) if with_intermediates else tuple(outs)


def load_case(name):
    from depth_from_motion_b200 import synthetic as syn
    seed, b, h, w = CASES[name]
    img, sd = syn.make_liga_resnet_case(seed, h, w, b)
    gold = dict(np.load(os.path.join(GOLDEN, 'liga_resnet.npz')))
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
        print(name, 'fp32', check_against_fixture(name, liga_resnet_forward(sd, img)))
        outs = liga_resnet_forward(fp64_params(sd), img.double())
        print(name, 'fp64', check_against_fixture(name, outs))


def test_mirror_state_dict_matches_reference():
    from depth_from_motion_b200 import modules
    gold = dict(np.load(os.path.join(GOLDEN, 'liga_resnet.npz')))
    sd = modules.LIGAResNet(**BACKBONE_CFG).state_dict()
    assert list(sd) == list(gold['state_keys'])
    assert [','.join(str(n) for n in v.shape) for v in sd.values()] == list(gold['state_shapes'])
    assert len(sd) == 204 and sum(v.numel() for v in sd.values()) == 4014562
    _, ref_sd, _, _ = load_case('small')
    modules.LIGAResNet(**BACKBONE_CFG).load_state_dict(ref_sd, strict=True)


def test_kitti_config_builds_liga_resnet():
    """The KITTI config's `backbone` (as registry.Config parsed it) builds the mirror through the
    local BACKBONES registry."""
    from depth_from_motion_b200 import modules, registry
    cfg = REFERENCE_IO['configs']['dfm_r34_1x8_kitti-3d-3class.py']['backbone']
    m = registry.build_backbone(dict(cfg))
    assert isinstance(m, modules.LIGAResNet)
    assert m.dilations == (1, 1, 2, 4) and m.strides == (1, 2, 1, 1)
    from oracle.ref_loader import REFERENCE_ROOT
    ref = os.path.join(REFERENCE_ROOT, 'configs', 'dfm', 'dfm_r34_1x8_kitti-3d-3class.py')
    if os.path.isfile(ref):
        direct = registry.Config.fromfile(ref).model['backbone']
        assert isinstance(registry.build_backbone(dict(direct)), modules.LIGAResNet)


@pytest.mark.parametrize('change', [
    dict(depth=18), dict(depth=50), dict(strides=(1, 2, 2, 2)), dict(dilations=(1, 1, 1, 1)),
    dict(num_channels_factor=(1, 2, 4, 8)), dict(num_channels_factor=None),
    dict(with_max_pool=True), dict(block_with_final_relu=True), dict(deep_stem=True),
    dict(avg_down=True), dict(dcn=dict(type='DCNv2'), stage_with_dcn=(False, False, True, True)),
    dict(plugins=[dict(cfg=dict(type='ContextBlock'), position='after_conv3')]),
    dict(norm_cfg=dict(type='GN', num_groups=32)),
    # the config's commented "sem" variant
    dict(strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), block_with_final_relu=True,
         norm_eval=True)])
def test_unsupported_options_raise(change):
    from depth_from_motion_b200 import modules
    with pytest.raises(NotImplementedError):
        modules.LIGAResNet(**dict(BACKBONE_CFG, **change))


def test_input_validation_before_any_launch():
    from depth_from_motion_b200 import modules
    m = modules.LIGAResNet(**BACKBONE_CFG).eval()
    for bad in (torch.zeros(3, 32, 32), torch.zeros(1, 4, 32, 32), torch.zeros(1, 1, 32, 32),
                torch.zeros(1, 3, 0, 32)):
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
    m = modules.LIGAResNet(**BACKBONE_CFG)
    full = {'backbone.' + k: v for k, v in sd.items()}
    full['backbone_stereo.foo'] = torch.zeros(1)
    full['neck.rpnconv.0.conv.weight'] = torch.zeros(1)
    res = checkpoint.load_hot_path({'state_dict': full}, img_backbone=m)
    assert not res['backbone'].missing_keys and not res['backbone'].unexpected_keys
    assert torch.equal(m.state_dict()['layer3.2.conv1.weight'], sd['layer3.2.conv1.weight'])
    parts = checkpoint.hot_path_state_dicts({'state_dict': full})
    assert list(parts['backbone_stereo']) == ['foo'] and 'foo' not in parts['backbone']
    m2 = modules.LIGAResNet(**BACKBONE_CFG)
    liga = {'model_state': {'backbone_3d.feature_backbone.' + k: v for k, v in sd.items()}}
    liga['model_state']['backbone_3d.cost_conv.0.weight'] = torch.zeros(1)
    checkpoint.load_hot_path(liga, img_backbone=m2)
    assert torch.equal(m2.state_dict()['layer4.2.bn2.running_var'], sd['layer4.2.bn2.running_var'])
    assert 'cost_conv.0.weight' in checkpoint.hot_path_state_dicts(liga)['backbone_stereo']
    with pytest.raises(KeyError, match='"backbone."'):
        checkpoint.load_hot_path({'state_dict': {'backbone_stereo.x': torch.zeros(1)}},
                                 img_backbone=modules.LIGAResNet(**BACKBONE_CFG))


def test_descriptor_matches_header():
    from depth_from_motion_b200 import capi
    src = open(HEADER).read()
    body = re.search(r'typedef struct dfm_liga_resnet_desc \{(.*?)\} dfm_liga_resnet_desc_t;',
                     src, re.S).group(1)
    fields = re.findall(r'int (\w+);', body)
    assert fields == [f for f, _ in capi.LigaResNetDesc._fields_]
    for fn in ('create', 'destroy', 'set_param', 'missing_params', 'forward', 'debug_tensor'):
        assert f'dfm_liga_resnet_{fn}' in capi.SYMBOLS
        assert f'dfm_liga_resnet_{fn}(' in src


def test_output_sizes_follow_pytorch():
    from depth_from_motion_b200 import modules
    for h, w in ((384, 1248), (70, 134), (71, 1), (1, 3)):
        ref = F.conv2d(torch.zeros(1, 1, h, w), torch.zeros(1, 1, 7, 7), None, 2, 3)
        ref2 = F.conv2d(ref, torch.zeros(1, 1, 3, 3), None, 2, 1)
        assert modules.LIGAResNet.output_sizes(h, w) == (tuple(ref.shape[2:]), tuple(ref2.shape[2:]))


# --- per-layer error model: bf16-split emulation of a conv with stride / padding / dilation ---
def conv64(x, w, stride=1, pad=None, dil=1):
    k = w.shape[-1]
    pad = (k // 2) * dil if pad is None else pad
    return F.conv2d(x, w, None, stride, pad, dil)


def emulated(x, w, **g):
    xh, xl = LC.split16(x)
    wh, wl = LC.split16(w)
    a, b, c = conv64(xh, wh, **g), conv64(xl, wh, **g), conv64(xh, wl, **g)
    return a + b + c, a + c, a + b


def layer_classes(sd, img):
    """(label, input, weight, geometry) of one layer of each new class: K = 147 (stem), 576
    (layer1), 1152 (layer2.1.conv1, and dilated layer3.0.conv1 / layer4.0.conv1), 64
    (downsample), fp64."""
    p = fp64_params(sd)
    with torch.no_grad():
        _, mid = liga_resnet_forward(p, img.double(), with_intermediates=True)
    return [('stem', img.double(), p['conv1.weight'], dict(stride=2, pad=3)),
            ('layer1.0.conv1', mid['layer1.0.in'], p['layer1.0.conv1.weight'], {}),
            ('layer2.1.conv1', mid['layer2.1.in'], p['layer2.1.conv1.weight'], {}),
            ('layer3.0.conv1', mid['layer3.0.in'], p['layer3.0.conv1.weight'], dict(dil=2)),
            ('layer4.0.conv1', mid['layer4.0.in'], p['layer4.0.conv1.weight'], dict(dil=4)),
            ('layer2.0.downsample', mid['layer2.0.in'], p['layer2.0.downsample.0.weight'],
             dict(stride=2, pad=0))]


def test_bound_separates_lost_term_cpu():
    img, sd, _, _ = load_case('small')
    for label, x, w, g in layer_classes(sd, img):
        ref = conv64(x, w, **g)
        e3, e2 = LC.norm_errors(emulated(x, w, **g), ref)
        k = w.shape[1] * w.shape[2] * w.shape[3]
        bound = layer_bound(e3, k, FLOOR_C)
        print(f'{label}: K {k} e3 {e3:.2e} e2 {e2:.2e} bound {bound:.2e} e2/bound {e2 / bound:.1f}')
        assert SEPARATION * bound <= e2, (label, bound, e2)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def make_backbone(sd, impl='auto'):
    from depth_from_motion_b200 import modules
    m = modules.LIGAResNet(**BACKBONE_CFG, conv_impl=impl)
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
    # 31 of the 33 convs are 3x3 stride 1: all on tensor cores under auto
    assert tc == (31 if impl == 'auto' else 0), tc
    print(name, impl, check_against_fixture(name, outs))


WHOLE_CASES = {'kitti': (61, 1, 384, 1248), 'crop_pair': (62, 2, 320, 1280),
               'odd': (52, 1, 70, 134), 'tiny': (63, 1, 12, 20)}


@pytest.mark.gpu
@pytest.mark.parametrize('impl', ['auto', 'simt'])
@pytest.mark.parametrize('case', list(WHOLE_CASES))
def test_whole_module_vs_fp64(case, impl):
    from depth_from_motion_b200 import synthetic as syn
    seed, b, h, w = WHOLE_CASES[case]
    img, sd = syn.make_liga_resnet_case(seed, h, w, b)
    m = make_backbone(sd, impl)
    with torch.no_grad():
        outs = m(img.cuda())
        ref = liga_resnet_forward(fp64_params(sd, 'cuda'), img.cuda().double())
    for lvl, (o, r) in enumerate(zip(outs, ref)):
        assert o.shape == r.shape
        print(case, impl, lvl, assert_close(o, r, f'{case} {impl} out{lvl}'))


def _shell(n, tile, d):
    """Output indices beside a tile seam (both sides), within d of either border, first / last."""
    i = torch.arange(n)
    sel = (i < max(d, 1)) | (i >= n - max(d, 1))
    if tile:
        sel |= (i % tile == 0) | (i % tile == tile - 1)
    return sel


class LayerChecker:
    """One row per conv: the GPU's raw output against fp64 from the GPU's own input, the bound
    max(6 e3, 8 sqrt(K) 2^-24) (the accumulation floor alone for CUDA-core layers), that bound
    >= 3x below the lost-term error e2, and the element-wise form on the tile / border shell of
    every image."""

    def __init__(self):
        self.rows, self.failures, self.checked = [], [], set()

    def conv(self, label, got, x, w, cls, tc, d=1, **g):
        ref = conv64(x, w, dil=d, **g)
        ys = emulated(x, w, dil=d, **g)
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
            sc = conv64(x.abs(), w.abs(), dil=d, **g)
            hh, ww = got.shape[2:]
            m = _shell(hh, TILE[0], d)[:, None] | _shell(ww, TILE[1], d)[None, :]
            m = m.to(got.device)
            sel = [t.movedim(1, -1)[:, m] for t in (got, ref) + tuple(ys) + (sc,)]
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
        self.rows.append(dict(layer=label, cls='block', err=e, bound=tol))
        if e > tol:
            self.failures.append((label, e, tol))

    def report(self, case):
        nan = float('nan')
        for r in self.rows:
            print(f"{case} | {r['layer']} | {r['cls']} | {r['err']:.2e} | {r['bound']:.2e} | "
                  f"{r.get('e3', nan):.2e} | {r.get('e2', nan):.2e} || {r.get('shell', nan):.2e} | "
                  f"{r.get('shell_bound', nan):.2e} | {r.get('shell_e2', nan):.2e}")


def run_layers(seed, b, h, w, impl='auto'):
    from depth_from_motion_b200 import synthetic as syn
    from tests.test_stage_layers import profiled
    img, sd = syn.make_liga_resnet_case(seed, h, w, b)
    m = make_backbone(sd, impl)
    img = img.cuda()
    _, report = profiled(lambda: m(img))
    p = fp64_params(sd, 'cuda')
    (h2, w2), (h4, w4) = m.output_sizes(h, w)
    ck = LayerChecker()

    def dbg(name, hh, ww, c):
        return m.debug_tensor(name, (b, hh, ww, c)).permute(0, 3, 1, 2).double()

    def folded(x, prefix, relu):
        s = p[prefix + '.weight'] / torch.sqrt(p[prefix + '.running_var'] + 1e-5)
        sh = (p[prefix + '.bias'] - p[prefix + '.running_mean'] * s).float().double()
        y = x * s.float().double()[:, None, None] + sh[:, None, None]
        return F.relu(y) if relu else y

    def cls_of(kind, cin, cout, k, s, d, hh, ww):
        return f'{kind}<{cin}->{cout},k{k},s{s},d{d}'

    tc_on = impl != 'simt'
    stem = dbg('stem', h2, w2, 64)
    ck.conv('stem', stem, img.double(), p['conv1.weight'],
            'resnet_stem<3->64,k7,s2', False, stride=2, pad=3)
    x = folded(stem, 'bn1', True)
    for name, s, j, stride, d in blocks():
        c = STAGES[s][1]
        cin = 64 if (s == 1 and j == 0) else c
        hh, ww = (h2, w2) if s == 0 else (h4, w4)
        tc1 = tc_on and stride == 1
        kind1 = 'resnet_conv_tc' if tc1 else 'resnet_conv_simt'
        r1 = dbg(name + '.conv1', hh, ww, c)
        ck.conv(name + '.conv1', r1, x, p[name + '.conv1.weight'],
                cls_of(kind1, cin, c, 3, stride, d, hh, ww), tc1, d=d, stride=stride)
        identity = x
        if stride != 1:
            rd = dbg(name + '.downsample', hh, ww, c)
            ck.conv(name + '.downsample', rd, x, p[name + '.downsample.0.weight'],
                    cls_of('resnet_conv_simt', cin, c, 1, 2, 1, hh, ww), False, stride=2, pad=0)
            identity = folded(rd, name + '.downsample.1', False)
        a1 = folded(r1, name + '.bn1', True)
        kind2 = 'resnet_conv_tc' if tc_on else 'resnet_conv_simt'
        r2 = dbg(name + '.conv2', hh, ww, c)
        ck.conv(name + '.conv2', r2, a1, p[name + '.conv2.weight'],
                cls_of(kind2, c, c, 3, 1, 1, hh, ww), tc_on)
        out = dbg(name, hh, ww, c)
        ck.elementwise(name, out, folded(r2, name + '.bn2', False) + identity)
        x = out
    launched = {k.split('>@')[0] for k in report if k.startswith('resnet_conv_tc<')}
    if launched - ck.checked:
        ck.failures.append(('tensor-core classes launched but not compared',
                            sorted(launched - ck.checked)))
    ck.report(f'liga_resnet {b}x{h}x{w} {impl}')
    print('CLASSES', ' '.join(sorted(report)))
    return ck, launched


@pytest.mark.gpu
def test_layers_vs_fp64_kitti_shape():
    ck, launched = run_layers(64, 1, 384, 1248)
    assert not ck.failures, ck.failures
    dils = {c.split(',d')[-1] for c in launched}
    assert dils == {'1', '2', '4'}, launched


@pytest.mark.gpu
def test_layers_vs_fp64_batch_odd():
    """Two ragged images in one call: tiles never straddle images, first / last cells of each."""
    ck, _ = run_layers(65, 2, 70, 134)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_layers_vs_fp64_simt():
    ck, launched = run_layers(66, 1, 70, 134, impl='simt')
    assert not launched
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_backbone_feeds_spp_neck():
    """Native LIGAResNet -> native SPPUNetNeck at 384 x 1248 against the restated chain."""
    from depth_from_motion_b200 import synthetic as syn
    from tests.test_spp_neck import NECK_CFG, spp_unet_neck_forward
    from depth_from_motion_b200 import modules
    h, w = 384, 1248
    img, sd = syn.make_liga_resnet_case(67, h, w, 1)
    _, nsd = syn.make_spp_neck_case(68, h, w)
    bb = make_backbone(sd)
    neck = modules.SPPUNetNeck(**NECK_CFG)
    neck.load_state_dict(nsd, strict=True)
    neck = neck.cuda().eval()
    with torch.no_grad():
        feats = bb(img.cuda())
        stereo, sem = neck([img.cuda()] + list(feats))
        rf = liga_resnet_forward(fp64_params(sd, 'cuda'), img.cuda().double())
        rs, rsem = spp_unet_neck_forward(fp64_params(nsd, 'cuda'), [img.cuda().double()] + list(rf))
    print('stereo', assert_close(stereo, rs, 'stereo'), 'sem', assert_close(sem, rsem, 'sem'))


@pytest.mark.gpu
def test_c_api_errors_and_repeatability():
    from depth_from_motion_b200 import capi
    L = capi.lib()
    img, sd, _, (_, b, h, w) = load_case('odd')
    for bad in ((0, 20, 1, 0), (20, 20, 0, 0), (20, 20, 1, 7)):
        hd = ctypes.c_void_p()
        assert L.dfm_liga_resnet_create(ctypes.byref(capi.LigaResNetDesc(*bad)),
                                        ctypes.byref(hd)) == 1, bad
    hd = ctypes.c_void_p()
    assert L.dfm_liga_resnet_create(ctypes.byref(capi.LigaResNetDesc(h, w, b, capi.DFM_CONV_TC)),
                                    ctypes.byref(hd)) == 0
    keys = [k for k in sd if not k.endswith('num_batches_tracked')]
    assert L.dfm_liga_resnet_missing_params(hd) == len(keys) == 170

    def put(k, v, n=None):
        v = v.float().contiguous()
        return L.dfm_liga_resnet_set_param(hd, k.encode(), ctypes.c_void_p(v.data_ptr()),
                                           v.numel() if n is None else n)
    for k in keys[:-1]:
        assert put(k, sd[k]) == 0, k
    outs = [torch.empty(b, 64, 35, 67, device='cuda')] + \
        [torch.empty(b, 128, 18, 34, device='cuda') for _ in range(3)]
    arr = (ctypes.c_void_p * 4)(*[o.data_ptr() for o in outs])
    x = img.cuda().contiguous()
    assert L.dfm_liga_resnet_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 3
    assert put(keys[-1], sd[keys[-1]], 7) == 1
    assert put('layer5.0.conv1.weight', sd[keys[-1]]) == 1
    assert put(keys[-1], sd[keys[-1]]) == 0
    buf = torch.empty(b * 35 * 67 * 64, device='cuda')
    assert L.dfm_liga_resnet_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel(), None) == 3
    _, t0 = capi.launch_counters()
    assert L.dfm_liga_resnet_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 0
    capi.sync_check()
    _, t1 = capi.launch_counters()
    assert t1 - t0 == 31
    first = [o.clone() for o in outs]
    assert L.dfm_liga_resnet_forward(hd, ctypes.c_void_p(x.data_ptr()), arr, None) == 0
    capi.sync_check()
    assert all(torch.equal(a, o) for a, o in zip(first, outs))       # bitwise repeatable
    assert L.dfm_liga_resnet_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel(), None) == 0
    assert L.dfm_liga_resnet_debug_tensor(hd, b'stem', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel() - 1, None) == 1
    assert L.dfm_liga_resnet_debug_tensor(hd, b'layer9.0', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel(), None) == 1
    L.dfm_liga_resnet_destroy(hd)
    # a batch of two gives each image what a batch of one gives it
    m = make_backbone(sd)
    with torch.no_grad():
        two = m(torch.cat((img, img.flip(-1))).cuda())
        one = m(img.flip(-1).cuda())
    assert all(torch.equal(t[:1], f) for t, f in zip(two, first))
    assert all(torch.equal(t[1:], o) for t, o in zip(two, one))
    assert not math.isnan(float(two[3].sum()))
