"""SPPUNetNeck (necks/spp_unet_neck.py, shipped KITTI config) on CUDA: fixture parity against the
reference module, state_dict / registry / checkpoint plumbing, shape rejections, per-layer fp64
checks at the benchmarked 384 x 1248 input, and the neck feeding DfMBackbone through its
channels-last twin.

``spp_unet_neck_forward`` below is the fp32 / fp64 restatement of the reference forward that the
fixture (tests/golden/make_spp_neck_golden.py) checks; the GPU tests compare against it.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O
from tests import layer_check as LC
from tests.layer_check import SEPARATION, layer_bound
from tests.test_stage_layers import (BEV_TILE, EW_TOL, FLOOR_C, Checker, _cl, classes_of, fp64,
                                     profiled)
from tests.util import GOLDEN, assert_close

# must match tests/golden/make_spp_neck_golden.py
CASES = {'small': (41, 256, 512), 'odd': (42, 300, 536)}
EDGE_CASES = ('odd',)
N_SAMPLE = {'stereo': 4096, 'sem': 8192}
NECK_CFG = dict(in_channels=[3, 64, 128, 128, 128], start_level=2, sem_channels=[128, 32],
                stereo_channels=[32, 32], with_upconv=True, cat_img_feature=True,
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
POOLS = (64, 32, 16, 8)


# ---------------------------------------------------------------------------------------------
# fp32 / fp64 restatement of the reference forward
# ---------------------------------------------------------------------------------------------
def _bn(x, p, prefix):
    """Eval BatchNorm2d / SyncBatchNorm (conv_modules.py:22)."""
    return F.batch_norm(x, p[prefix + '.running_mean'], p[prefix + '.running_var'],
                        p[prefix + '.weight'], p[prefix + '.bias'], False, 0.0, 1e-5)


def spp_branch(p, f4, i):
    """spp_branches[i] (spp_unet_neck.py:35-46): AvgPool2d(s) (floor mode), 1x1 conv, GN, ReLU."""
    x = F.avg_pool2d(f4, POOLS[i], POOLS[i])
    x = F.conv2d(x, p[f'spp_branches.{i}.1.conv.weight'])
    return F.relu(O._gn2d(x, p, f'spp_branches.{i}.1.gn'))


def spp_unet_neck_forward(p, feats, with_intermediates=False):
    """SPPUNetNeck.forward (spp_unet_neck.py:93-119) with upconv_module.forward
    (conv_modules.py:63-69) for the shipped KITTI config.  Returns (stereo_feature,
    sem_feature[, dict of the branch maps before upsampling, concat, x0, x1])."""
    img, f1, f2, f3, f4 = feats
    size = tuple(f2.shape[2:])
    maps = [spp_branch(p, f4, i) for i in range(4)]
    ups = [F.interpolate(m, size, mode='bilinear', align_corners=True) for m in maps]
    cat = torch.cat((f2, f3, f4, *ups), 1)                                     # :104

    def convbn(x, name):
        return _bn(F.conv2d(x, p[f'upconv_module.{name}.0.weight'], None, 1, 1), p,
                   f'upconv_module.{name}.1')

    def up(x):
        return F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)
    x0 = F.relu(up(convbn(cat, 'conv.0')) + convbn(f1, 'redir.0'))
    x1 = F.relu(up(convbn(x0, 'conv.1')) + convbn(img, 'redir.1'))
    stereo = O.spp_unet_lastconv(p, x1)                                        # :112
    sem = F.relu(O._gn2d(F.conv2d(cat, p['rpnconv.0.conv.weight'], None, 1, 1), p, 'rpnconv.0.gn'))
    sem = F.relu(O._gn2d(F.conv2d(sem, p['rpnconv.1.conv.weight'], None, 1, 1), p, 'rpnconv.1.gn'))
    if with_intermediates:
        return stereo, sem, dict(maps=maps, cat=cat, x0=x0, x1=x1)
    return stereo, sem


def load_case(name):
    from depth_from_motion_b200 import synthetic as syn
    seed, h, w = CASES[name]
    feats, sd = syn.make_spp_neck_case(seed, h, w)
    gold = dict(np.load(os.path.join(GOLDEN, 'spp_neck.npz')))
    return feats, sd, gold, (seed, h, w)


def check_against_fixture(name, stereo, sem, maps=None):
    """stereo_feature and sem_feature at the stored seeded samples (and first / last rows and
    columns for the ragged-tile case), the branch maps in full."""
    feats, sd, gold, (seed, h, w) = load_case(name)
    worst = {}
    for what, t in (('stereo', stereo), ('sem', sem)):
        t = t[0].detach().cpu()
        th, tw = t.shape[1:]
        idx = np.random.RandomState(seed + (1000 if what == 'stereo' else 2000)).randint(
            0, 32 * th * tw, N_SAMPLE[what])
        parts = [('sample', t.reshape(-1)[torch.from_numpy(idx)])]
        if name in EDGE_CASES:
            parts += [('rows', t[:, [0, th - 1], :]), ('cols', t[:, :, [0, tw - 1]])]
        for part, got in parts:
            key = f'{name}_{what}_{part}'
            worst[f'{what}_{part}'] = assert_close(got, gold[key], key)
    if maps is not None:
        for i in range(4):
            worst[f'spp{POOLS[i]}'] = assert_close(maps[i][0].detach().cpu(),
                                                   gold[f'{name}_spp{i}'], f'{name} spp{i}')
    return worst


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(CASES))
def test_oracle_reproduces_fixture(name):
    feats, sd, gold, _ = load_case(name)
    sums = np.array([[f.double().sum().item(), f.double().abs().sum().item()] for f in feats])
    np.testing.assert_allclose(sums, gold[f'{name}_feat_sums'], rtol=1e-9)
    np.testing.assert_allclose(sum(v.double().abs().sum().item() for v in sd.values()),
                               gold[f'{name}_w_abs'], rtol=1e-9)
    with torch.no_grad():
        stereo, sem, mid = spp_unet_neck_forward(sd, feats, with_intermediates=True)
    print(name, check_against_fixture(name, stereo, sem, mid['maps']))


def test_mirror_state_dict_matches_reference():
    from depth_from_motion_b200 import modules
    gold = dict(np.load(os.path.join(GOLDEN, 'spp_neck.npz')))
    sd = modules.SPPUNetNeck(**NECK_CFG).state_dict()
    assert list(sd) == list(gold['state_keys'])
    assert [','.join(str(n) for n in v.shape) for v in sd.values()] == list(gold['state_shapes'])
    assert len(sd) == 46 and sum(v.numel() for v in sd.values()) == 1005796
    _, ref_sd, _, _ = load_case('small')
    modules.SPPUNetNeck(**NECK_CFG).load_state_dict(ref_sd, strict=True)


def test_kitti_config_builds_spp_neck():
    from depth_from_motion_b200 import modules, registry
    m = registry.build_neck(dict(type='SPPUNetNeck', **NECK_CFG))
    assert isinstance(m, modules.SPPUNetNeck)
    assert m.cat_img_feature and m.sem_channels == [128, 32]   # detectors/dfm.py:55-64
    with pytest.raises(AssertionError):
        modules.SPPUNetNeck(**dict(NECK_CFG, spp_channel=64))


def test_load_hot_path_loads_img_neck():
    from depth_from_motion_b200 import checkpoint, modules
    _, sd, _, _ = load_case('small')
    m = modules.SPPUNetNeck(**NECK_CFG)
    full = {'neck.' + k: v for k, v in sd.items()}
    full['neck_3d.foo'] = torch.zeros(1)
    full['neck_2d.lateral.weight'] = torch.zeros(1)
    res = checkpoint.load_hot_path({'state_dict': full}, img_neck=m)
    assert not res['neck'].missing_keys and not res['neck'].unexpected_keys
    assert torch.equal(m.state_dict()['rpnconv.0.conv.weight'], sd['rpnconv.0.conv.weight'])
    m2 = modules.SPPUNetNeck(**NECK_CFG)
    liga = {'model_state': {'backbone_3d.feature_neck.' + k: v for k, v in sd.items()}}
    checkpoint.load_hot_path(liga, img_neck=m2)
    assert torch.equal(m2.state_dict()['lastconv.1.weight'], sd['lastconv.1.weight'])
    with pytest.raises(KeyError, match='"neck."'):
        checkpoint.load_hot_path({'state_dict': {'neck_3d.x': torch.zeros(1)}},
                                 img_neck=modules.SPPUNetNeck(**NECK_CFG))


def _feats(h, w, b=1, f1_hw=None):
    f1_hw = f1_hw or (h // 2, w // 2)
    return [torch.zeros(b, 3, h, w), torch.zeros(b, 64, *f1_hw)] + \
        [torch.zeros(b, 128, h // 4, w // 4)] * 3


@pytest.mark.parametrize('h,w,f1_hw', [(264, 392, None), (240, 1248, None),
                                       (256, 512, (130, 256)), (258, 512, None)])
def test_shape_rejections(h, w, f1_hw):
    """264 x 392: the 64-pool leaves 1 cell (GroupNorm raises); 240 x 1248: 0 rows (AvgPool2d
    raises); f1 not twice f2, or an image that is not a multiple of 4: the adds fail."""
    from depth_from_motion_b200 import modules
    with pytest.raises(ValueError):
        modules.SPPUNetNeck.check_shapes(_feats(h, w, f1_hw=f1_hw))
    modules.SPPUNetNeck.check_shapes(_feats(256, 520))


def _layer_inputs(sd, feats):
    """(label, input, weight, k) of the five tensor-core layer classes and lastconv, fp64."""
    p = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
    f = [t.double() for t in feats]
    with torch.no_grad():
        _, _, mid = spp_unet_neck_forward(p, f, with_intermediates=True)
        rpn0 = F.conv2d(mid['cat'], p['rpnconv.0.conv.weight'], None, 1, 1)
        a1 = F.relu(O._gn2d(rpn0, p, 'rpnconv.0.gn'))
    return [('conv0', mid['cat'], p['upconv_module.conv.0.0.weight']),
            ('rpn0', mid['cat'], p['rpnconv.0.conv.weight']),
            ('redir0', f[1], p['upconv_module.redir.0.0.weight']),
            ('conv1', mid['x0'], p['upconv_module.conv.1.0.weight']),
            ('rpn1', a1, p['rpnconv.1.conv.weight']),
            ('lastconv', mid['x1'], p['lastconv.0.conv.weight'])]


def test_bound_separates_lost_term_cpu():
    feats, sd, _, _ = load_case('small')
    for label, x, w in _layer_inputs(sd, feats):
        ref = LC.conv_planes(x, w)
        e3, e2 = LC.emulate(x, w, ref)
        k = LC.k_of(x.shape[1], nd=2)
        bound = layer_bound(e3, k, FLOOR_C)
        print(f'{label}: e3 {e3:.2e} e2 {e2:.2e} bound {bound:.2e} e2/bound {e2 / bound:.1f}')
        assert SEPARATION * bound <= e2, (label, bound, e2)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def make_neck(sd, impl='auto'):
    from depth_from_motion_b200 import modules
    m = modules.SPPUNetNeck(**NECK_CFG, conv_impl=impl)
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
    feats, sd, _, _ = load_case(name)
    m = make_neck(sd, impl)
    fc = [f.cuda() for f in feats]
    with torch.no_grad():
        m(fc)
        (stereo, sem), tc = _tc_count(lambda: m(fc))
        maps = [m.debug_tensor(f'spp{s}', (shape[2], shape[3], 32)).permute(2, 0, 1)[None]
                for s, shape in zip(POOLS, (spp_branch(sd, feats[4], i).shape
                                            for i in range(4)))]
    # five 3x3 convs on the 2-D layer driver plus lastconv: all on the tensor cores under auto
    assert tc == (6 if impl == 'auto' else 0), tc
    print(name, impl, check_against_fixture(name, stereo, sem, maps))


def run_layers(sd, feats, impl='auto'):
    """One profiled forward; every conv against fp64 from the GPU's own inputs, every non-GEMM
    kernel element-wise."""
    m = make_neck(sd, impl)
    fc = [f.cuda() for f in feats]
    (stereo, sem), report = profiled(lambda: m(fc))
    h, w = feats[0].shape[2:]
    h2, w2, h4, w4 = h // 2, w // 2, h // 4, w // 4
    p = fp64({k: v for k, v in sd.items() if v.is_floating_point()}, 'cuda')
    f = [t.cuda().double() for t in feats]
    simt = impl == 'simt'
    ck = Checker(f'spp_neck {h}x{w}' + (' [simt]' if simt else ''))

    def dbg(name, *shape):
        return _cl(m.debug_tensor(name, shape))

    def conv(label, cin, cout, hw, x, wt):
        raw = dbg(label, *hw, cout)
        kind, dims = ('conv_tc', (1,) + hw) if label == 'lastconv' else ('conv2d_tc', hw + (1,))
        cls = classes_of(report, (kind,), cin, cout, ('s1',), dims)
        cls += classes_of(report, ('conv2d_simt', 'conv_simt'), cin, cout, ('s1',), (1,) + hw)
        tc = any('_tc' in c for c in cls)
        assert tc != simt, (label, cls)
        ck.conv(label, raw, x, wt, cls, LC.k_of(cin, nd=2),
                tiles=BEV_TILE if tc and label != 'lastconv' else None, simt=not tc)
        return raw

    def folded(x, prefix):
        s = p[prefix + '.weight'] / torch.sqrt(p[prefix + '.running_var'] + 1e-5)
        sh = (p[prefix + '.bias'] - p[prefix + '.running_mean'] * s).float().double()
        return x * s.float().double()[:, None, None] + sh[:, None, None]

    def up(x):
        return F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)

    # SPP: pools, branches (GN amplifies the fp32 rounding of the 1x1 conv by gamma / std: the
    # element-wise bound carries that factor), concat
    maps = []
    for i, s in enumerate(POOLS):
        ph, pw = h4 // s, w4 // s
        pool = dbg(f'pool{s}', ph, pw, 128)
        ck.elementwise(f'pool{s}', pool, F.avg_pool2d(f[4], s, s), cls='spp_pool')
        br = dbg(f'spp{s}', ph, pw, 32)
        wt = p[f'spp_branches.{i}.1.conv.weight']
        raw = F.conv2d(pool, wt)
        var = raw.var(dim=(2, 3), unbiased=False)[0]
        ref = F.relu(O._gn2d(raw, p, f'spp_branches.{i}.1.gn'))
        amp = (p[f'spp_branches.{i}.1.gn.weight'].abs() / torch.sqrt(var + 1e-5))[:, None, None]
        tol = LC.acc_floor(128, FLOOR_C) * F.conv2d(pool.abs(), wt.abs()) * amp * 2 + \
            1e-6 * float(ref.abs().max())
        ratio = float(((br - ref).abs() / tol).max())
        ck.rows.append(dict(layer=f'spp{s}', cls='spp_branch', err=ratio, bound=1.0))
        if ratio > 1.0:
            ck.failures.append((f'spp{s}', ratio))
        maps.append(br)
    cat = dbg('concat', h4, w4, 512)
    ups = [F.interpolate(mp, (h4, w4), mode='bilinear', align_corners=True) for mp in maps]
    # fp32 source coordinates (scale * index) against exact ones: up to ~1e-7 x 38 cells of
    # position times the neighbour difference; 3e-5 of the map's max
    ck.elementwise('concat', cat, torch.cat((f[2], f[3], f[4], *ups), 1), tol=3e-5,
                   cls='spp_concat')
    # convs and merges in forward order
    r_c0 = conv('conv0', 512, 64, (h4, w4), cat, p['upconv_module.conv.0.0.weight'])
    r_rd0 = conv('redir0', 64, 64, (h2, w2), f[1], p['upconv_module.redir.0.0.weight'])
    x0 = dbg('x0', h2, w2, 64)
    ck.elementwise('x0', x0, F.relu(up(folded(r_c0, 'upconv_module.conv.0.1')) +
                                    folded(r_rd0, 'upconv_module.redir.0.1')),
                   cls='upconv_merge')
    r_c1 = conv('conv1', 64, 32, (h2, w2), x0, p['upconv_module.conv.1.0.weight'])
    x1 = dbg('x1', h, w, 32)
    rd1 = F.conv2d(f[0], p['upconv_module.redir.1.0.weight'], None, 1, 1)
    ck.elementwise('x1', x1, F.relu(up(folded(r_c1, 'upconv_module.conv.1.1')) +
                                    folded(rd1, 'upconv_module.redir.1.1')),
                   cls='upconv_merge_img')
    r_last = conv('lastconv', 32, 32, (h, w), x1, p['lastconv.0.conv.weight'])
    ck.elementwise('stereo', stereo.double(),
                   F.conv2d(F.relu(O._gn2d(r_last, p, 'lastconv.0.gn')), p['lastconv.1.weight']),
                   cls='stereo_tail')
    r_p0 = conv('rpn0', 512, 128, (h4, w4), cat, p['rpnconv.0.conv.weight'])
    r_p1 = conv('rpn1', 128, 32, (h4, w4), F.relu(O._gn2d(r_p0, p, 'rpnconv.0.gn')),
                p['rpnconv.1.conv.weight'])
    ck.elementwise('sem', sem.double(), F.relu(O._gn2d(r_p1, p, 'rpnconv.1.gn')), cls='bev_emit')
    for tag in ('spp_pool', 'spp_branch', 'spp_concat', 'upconv_merge', 'upconv_merge_img'):
        if tag not in report:
            ck.failures.append(('no profile record', tag))
    ck.report(report)
    return ck


@pytest.mark.gpu
def test_layers_vs_fp64_kitti_shape():
    from depth_from_motion_b200 import synthetic as syn
    feats, sd = syn.make_spp_neck_case(43, 384, 1248)
    ck = run_layers(sd, feats)
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_layers_vs_fp64_simt():
    feats, sd, _, _ = load_case('odd')
    ck = run_layers(sd, feats, impl='simt')
    assert not ck.failures, ck.failures


@pytest.mark.gpu
def test_neck_feeds_backbone_channels_last():
    """cur and prev images through SPPUNetNeck, then DfMBackbone on the channels-last twins;
    against the oracle neck followed by the oracle backbone on NCHW."""
    from depth_from_motion_b200 import capi, modules
    from depth_from_motion_b200 import synthetic as syn
    h, w, d = 256, 512, 8
    cur, sd = syn.make_spp_neck_case(44, h, w)
    prev, _ = syn.make_spp_neck_case(45, h, w)
    _, _, metas, params = syn.make_kitti_pair(46, h, w, d)
    cfg = syn.depth_cfg_for(d)
    neck = make_neck(sd)
    bb = modules.DfMBackbone(in_channels=32, depth_cfg=cfg).cuda().eval()
    bb.load_state_dict(params, strict=True)
    bb.downsampled_depth = O.downsampled_depth(cfg)
    with torch.no_grad():
        rc, rsc = spp_unet_neck_forward(sd, cur)
        rp, _ = spp_unet_neck_forward(sd, prev)
        ref = O.dfm_backbone_forward(params, rc, rp, metas, cfg)
        sc, semc = neck([f.cuda() for f in cur])
        sp, _ = neck([f.cuda() for f in prev])
        assert sc._dfm_cl is not None and sp._dfm_cl is not None
        assert torch.equal(sc._dfm_cl.permute(2, 0, 1)[None], sc)
        bb(sc, sp, metas)                                    # build the handle
        capi.sync_check()
        l0, _ = capi.launch_counters()
        out = bb(sc, sp, metas)
        capi.sync_check()
        l1, _ = capi.launch_counters()
        out_nchw = bb(sc.clone(), sp.clone(), metas)         # no twin: two transposes
        capi.sync_check()
        l2, _ = capi.launch_counters()
    assert (l2 - l1) - (l1 - l0) == 2, (l1 - l0, l2 - l1)
    for a, b in zip(out, out_nchw):
        assert torch.equal(a, b)
    errs = {}
    for label, a, b in (('cost', out[0], ref[0]), ('stereo', out[1], ref[1]),
                        ('mono', out[2], ref[2]), ('sem', semc, rsc)):
        errs[label] = float((a.cpu().double() - b.double()).abs().max() / b.double().abs().max())
        assert errs[label] < 1e-3, (label, errs[label])
    print('neck -> backbone rel errs', errs)


@pytest.mark.gpu
def test_batch_two_repeatable():
    feats, sd, _, _ = load_case('odd')
    m = make_neck(sd)
    one = [f.cuda() for f in feats]
    with torch.no_grad():
        s1, e1 = m(one)
        s1b, e1b = m(one)
        assert torch.equal(s1, s1b) and torch.equal(e1, e1b)   # bitwise repeatable
        two = [torch.cat((f, f.flip(-1)), 0).cuda() for f in feats]
        s2, e2 = m(two)
        sf, ef = m([f.flip(-1).cuda() for f in feats])
    assert not hasattr(s2, '_dfm_cl')
    assert torch.equal(s2[:1], s1) and torch.equal(e2[:1], e1)
    assert torch.equal(s2[1:], sf) and torch.equal(e2[1:], ef)


class _Handle:
    def __init__(self, h, w, impl):
        from depth_from_motion_b200 import capi
        self.L, self.h = capi.lib(), ctypes.c_void_p()
        self.rc = self.L.dfm_spp_neck_create(h, w, impl, ctypes.byref(self.h))

    def set(self, k, v, n=None):
        v = v.detach().float().contiguous()
        return self.L.dfm_spp_neck_set_param(self.h, k.encode(), ctypes.c_void_p(v.data_ptr()),
                                             v.numel() if n is None else n)

    def forward(self, feats, cl, nchw, sem):
        ptr = [ctypes.c_void_p(t.data_ptr()) if t is not None else None
               for t in list(feats) + [cl, nchw, sem]]
        return self.L.dfm_spp_neck_forward(self.h, *ptr, None)

    def close(self):
        self.L.dfm_spp_neck_destroy(self.h)


@pytest.mark.gpu
def test_canary_tails_untouched():
    from depth_from_motion_b200 import capi
    feats, sd, _, (_, h, w) = load_case('odd')
    hd = _Handle(h, w, capi.DFM_CONV_AUTO)
    assert hd.rc == 0
    for k, v in sd.items():
        if not k.endswith('num_batches_tracked'):
            assert hd.set(k, v) == 0, k
    canary = 1234.5
    n_st, n_sem, pad = 32 * h * w, 32 * (h // 4) * (w // 4), 4096
    cl, nchw, sem = (torch.full((n + pad,), canary, device='cuda') for n in (n_st, n_st, n_sem))
    fc = [f.cuda().contiguous() for f in feats]
    assert hd.forward(fc, cl, nchw, sem) == 0
    capi.sync_check()
    for t, n in ((cl, n_st), (nchw, n_st), (sem, n_sem)):
        assert bool((t[n:] == canary).all())
        assert not bool((t[:n] == canary).any())
    ref, _ = make_neck(sd)(fc)
    assert torch.equal(nchw[:n_st].view(1, 32, h, w), ref)
    hd.close()


@pytest.mark.gpu
def test_errors():
    from depth_from_motion_b200 import capi, modules
    feats, sd, _, (_, h, w) = load_case('small')
    for bad in ((264, 392), (240, 1248), (258, 512), (256, 510)):
        hb = _Handle(*bad, capi.DFM_CONV_AUTO)
        assert hb.rc == 1, bad                                     # DFM_ERR_INVALID
    hd = _Handle(h, w, capi.DFM_CONV_TC)
    assert hd.rc == 0
    keys = [k for k in sd if not k.endswith('num_batches_tracked')]
    assert len(keys) == 42
    for k in keys[:-1]:
        assert hd.set(k, sd[k]) == 0, k
    fc = [f.cuda().contiguous() for f in feats]
    out = [torch.empty(32 * h * w, device='cuda'), None,
           torch.empty(32 * (h // 4) * (w // 4), device='cuda')]
    assert hd.L.dfm_spp_neck_missing_params(hd.h) == 1
    assert hd.forward(fc, *out) == 3                               # DFM_ERR_STATE
    assert hd.set(keys[-1], sd[keys[-1]], 7) == 1                  # wrong element count
    assert hd.set('rpnconv.2.conv.weight', sd[keys[-1]]) == 1      # unknown key
    assert hd.set(keys[-1], sd[keys[-1]]) == 0
    # debug hook before any forward: nothing written yet
    buf = torch.empty(64 * 64 * 128, device='cuda')
    assert hd.L.dfm_spp_neck_debug_tensor(hd.h, b'conv0', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel(), None) == 3
    # conv_impl='tc': every conv of the neck has a tensor-core kernel, so it runs and launches
    # only tensor-core convs (a layer without one would fail with DFM_ERR_INVALID)
    _, t0 = capi.launch_counters()
    assert hd.forward(fc, *out) == 0
    capi.sync_check()
    _, t1 = capi.launch_counters()
    assert t1 - t0 == 6
    assert hd.L.dfm_spp_neck_debug_tensor(hd.h, b'conv0', ctypes.c_void_p(buf.data_ptr()),
                                          buf.numel() - 1, None) == 1
    assert hd.L.dfm_spp_neck_debug_tensor(hd.h, b'conv0', ctypes.c_void_p(buf.data_ptr()),
                                          64 * 128 * 64, None) == 0
    hd.close()
    with pytest.raises(ValueError):
        modules.SPPUNetNeck(**NECK_CFG).cuda()(_gpu_feats(264, 392))


def _gpu_feats(h, w):
    return [torch.zeros(1, 3, h, w, device='cuda'), torch.zeros(1, 64, h // 2, w // 2, device='cuda')] + \
        [torch.zeros(1, 128, h // 4, w // 4, device='cuda')] * 3
