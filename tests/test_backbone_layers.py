"""Layer-by-layer parity of DfMBackbone's CUDA path against an fp64 reference.

The end-to-end tests hold the backbone outputs to the 1e-3 north-star bar.  That bar is far
above what one defective layer costs: DESIGN.md section 1 measures 7.9e-4 .. 3.1e-3 at the
logits for dropping ONE of the three bf16 product terms on one layer, and 1.6e-4 .. 4.2e-4 for a
TF32-like pass.  Here every conv of both towers is judged on its own instead:

* one forward of ``DfMBackbone(conv_impl='auto')``; its intermediates are read back through
  ``DfMBackbone.debug_tensor`` (``dfm_backbone_debug_tensor``);
* each layer's input is rebuilt in float64 from the GPU's OWN upstream raw outputs, with the
  GroupNorm statistics recomputed in float64 and GN / ReLU / residual applied exactly as
  ``oracle.dfm_oracle`` (``_tower``, ``hourglass``, ``_pred``) does;
* the layer's conv is run in float64 and compared with the GPU's raw output of that layer.

So errors do not carry over from earlier layers, wrong statistics show up in the consuming
layer, and every tile, window and z end of every kernel is checked directly.

Bounds come from emulation.  For each layer and input, ``e3`` is the error the kernels' 3-term
split ``x_hi w_hi + x_lo w_hi + x_hi w_lo`` (bf16 operand pairs) commits in exact accumulation,
``e2`` the smaller of the two 2-term variants (one lo term dropped).  A layer passes when its
error is below ``max(K_E3 * e3, fp32 accumulation floor)``, and that bound must stay at least
``SEPARATION`` times below ``e2``, so no bound can admit a lost term.  The CPU test
``test_bounds_separate_lost_term`` checks that separation on oracle inputs without a GPU.
The reference convs, the emulation and the bounds live in ``tests/layer_check.py``.

The shortened mono tower (D >= 48) computes 16 head, 8 interior and 16 tail planes at full
resolution (20 / 10 at the lower levels).  Its inputs are expanded to full depth with the phase
mapping of ``ZExpand`` (head planes map to themselves, interior planes repeat with period 4/s at
scale s, tail planes shift by (D - 40)/s), the statistics are computed on the expanded tensor,
and the computed planes are compared with the matching full planes; this checks the z-weighted
statistics sums of the epilogues directly.
"""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O
from tests import layer_check as LC
from tests import plane_sweep_check as PS
from tests.layer_check import SEPARATION, elementwise_errors, layer_bound

# ---------------------------------------------------------------------------------------------
# shapes (D, Ho = h/4 and Wo = w/4 are multiples of 4)
# ---------------------------------------------------------------------------------------------
CASES = {
    # Ho x Wo = 12 x 20: ragged 8 x 16 conv tiles on every level, odd 3 x 5 quarter resolution,
    # ragged 16-plane logits chunk and 14 x 6 logits tiles, D % 16 != 0 in the gate
    'ragged_48x80_d12': dict(seed=41, h=48, w=80, d=12),
    # kitti_aug-style flip + crop + scale (warp samples leave the image); shortened mono tower
    # with (D - 32) % 8 == 4, i.e. interior statistics weight 4.5
    'aug_64x112_d68': dict(seed=42, h=64, w=112, d=68, flip=True, crop=(10, 40), scale=1.03,
                           ori=(375, 1242, 3)),
    # the benchmarked shape: conv2 / conv4 on the K-outer kernel, full-size tile grids
    'bench_384x1248_d112': dict(seed=3, h=384, w=1248, d=112, ori=(370, 1224, 3), slabs=True),
    # the shipped KITTI config: D % 16 == 8 in the logits chunks and the gate at full width
    'kitti_320x1280_d72': dict(seed=21, h=320, w=1280, d=72, crop=(0, 55), ori=(375, 1242, 3),
                               slabs=True),
    # the gate's fallbacks, chosen by D alone (Ho * Wo is always a multiple of 16): at D = 120
    # gate_tile4's shared memory no longer fits, at D = 148 gate_persistent's neither
    'gate_persistent_48x80_d120': dict(seed=43, h=48, w=80, d=120),
    'gate_v1_48x80_d148': dict(seed=44, h=48, w=80, d=148),
}
# the cases the CPU bound-separation test evaluates with the oracle (the large ones are
# checked on the GPU, which also asserts the separation on the GPU's own layer inputs)
CPU_CASES = ('ragged_48x80_d12', 'aug_64x112_d68')

Z_HEAD, Z_MID = 16, 8   # tower_forward's kZHead / kZMid


def make_case(name):
    from depth_from_motion_b200 import synthetic as syn
    c = CASES[name]
    cur, prev, metas, params = syn.make_kitti_pair(
        c['seed'], c['h'], c['w'], c['d'], flip=c.get('flip', False),
        crop_offset=c.get('crop', (0, 0)), scale=c.get('scale', 1.0), ori_shape=c.get('ori'))
    return cur, prev, metas, params, syn.depth_cfg_for(c['d'])


def slabs_of(name):
    """Full-resolution z ranges compared: both z ends, the mono tower's interior planes
    [16, 24), and one interior slab.  Every slab is 4-aligned, so it maps onto whole planes of
    the two lower levels.  The K-outer kernel cuts D into 4-aligned windows of 4 planes: the
    8-aligned slabs end on window edges at half resolution, and the interior slab is offset
    by 4 planes so that it straddles a window seam at half and at quarter resolution."""
    d = CASES[name]['d']
    if not CASES[name].get('slabs'):
        return [(0, d)]
    mid = (d // 2) // 8 * 8 + 4
    return sorted({(0, 8), (16, 24), (mid, mid + 8), (d - 8, d)})


# ---------------------------------------------------------------------------------------------
# fp64 reference building blocks
# ---------------------------------------------------------------------------------------------
def _gn(x, p, prefix):
    return F.group_norm(x, 32, p[prefix + '.weight'], p[prefix + '.bias'], O.GN_EPS)


def geom(mode, z0, z1):
    """Geometry (tests/layer_check.py) of output planes [z0, z1) of conv3d(k3, p1, stride 1 | 2)
    ('s1' | 's2') or conv_transpose3d(k3, s2, p1, op1) ('t').  z0 must be even for 't'."""
    return dict(stride=2 if mode == 's2' else 1, transposed=mode == 't',
                region=((z0, z1), None, None))


def conv_planes(x, w, mode, z0, z1):
    return LC.conv_planes(x, w, **geom(mode, z0, z1))


def emulated_outputs(x, w, mode, z0, z1):
    return LC.emulated_outputs(x, w, **geom(mode, z0, z1))


def emulate(x, w, mode, z0, z1, ref):
    return LC.emulate(x, w, ref, **geom(mode, z0, z1))


def product_scale(x, w, mode, z0, z1):
    return LC.product_scale(x, w, **geom(mode, z0, z1))


def k_of(cin, mode):
    return LC.k_of(cin, mode == 't')


def tower_layers(vol, p, mono, fetch):
    """The convs of one tower in forward order, as (layer, input, weight, mode, level) with the
    input rebuilt in fp64 from fetch(name) -- the full-depth raw output of an upstream layer
    (dfm_backbone.py:175-197 + conv_modules.py:129-149 + dfm_backbone.py:118-128, i.e.
    oracle._tower / hourglass / _pred).  level = resolution divisor of the layer's OUTPUT."""
    sfx = '_mono' if mono else ''
    hg = ('hg_mono' if mono else 'hg_stereo') + '.0'
    pr = ('pred_mono' if mono else 'pred_stereo') + '.0'
    x0 = vol[:, :32] if mono else vol
    yield 'raw0', x0, p[f'dres0{sfx}.conv.weight'], 's1', 1
    a0 = F.relu(_gn(fetch('raw0'), p, f'dres0{sfx}.gn'))
    yield 'raw1', a0, p[f'dres1{sfx}.conv.weight'], 's1', 1
    cost0 = _gn(fetch('raw1'), p, f'dres1{sfx}.gn') + a0
    yield 'c1', cost0, p[f'{hg}.conv1.0.0.weight'], 's2', 2
    x = F.relu(_gn(fetch('c1'), p, f'{hg}.conv1.0.1'))
    yield 'c2', x, p[f'{hg}.conv2.0.weight'], 's1', 2
    pre = F.relu(_gn(fetch('c2'), p, f'{hg}.conv2.1'))
    yield 'c3', pre, p[f'{hg}.conv3.0.0.weight'], 's2', 4
    x = F.relu(_gn(fetch('c3'), p, f'{hg}.conv3.0.1'))
    yield 'c4', x, p[f'{hg}.conv4.0.0.weight'], 's1', 4
    x = F.relu(_gn(fetch('c4'), p, f'{hg}.conv4.0.1'))
    yield 'c5', x, p[f'{hg}.conv5.0.weight'], 't', 2
    post = F.relu(_gn(fetch('c5'), p, f'{hg}.conv5.1') + pre)
    yield 'c6', post, p[f'{hg}.conv6.0.weight'], 't', 1
    cur = cost0 + _gn(fetch('c6'), p, f'{hg}.conv6.1')
    yield 'cur', cur, None, None, 1          # not a conv: the materialised cur_cost
    yield 'p0', fetch('cur'), p[f'{pr}.0.conv.weight'], 's1', 1
    x = F.relu(_gn(fetch('p0'), p, f'{pr}.0.gn'))
    yield 'logit', x, p[f'{pr}.1.weight'], 's1', 1


def gate(logit, logit_mono, wagg):
    """dfm_backbone.py:130-141 on the two [1, 1, D, H, W] logit volumes."""
    cost = torch.cat((logit, logit_mono), dim=1).flatten(1, 2)
    w = F.conv2d(cost, wagg).unsqueeze(1).sigmoid()
    return w * logit + (1 - w) * logit_mono


def fp64_params(params, dev):
    return {k: torch.as_tensor(v).to(dev, torch.float64) for k, v in params.items()}


# ---------------------------------------------------------------------------------------------
# CPU: the bounds keep a lost product term out, at the test shapes
# ---------------------------------------------------------------------------------------------
LAYER_CLASS = {'raw0': 'dres0 (warp loader)', 'raw1': 'dres1', 'c1': 'conv1 s2 (cluster)',
               'c2': 'conv2', 'c3': 'conv3 s2 (K-slice)', 'c4': 'conv4',
               'c5': 'conv5 T', 'c6': 'conv6 T (2 terms)', 'p0': 'pred.0',
               'logit': 'pred.1 (logits)'}


@pytest.mark.parametrize('name', CPU_CASES)
def test_bounds_separate_lost_term(name):
    """On the oracle's own fp64 layer inputs: for every conv of both towers, the pass bound
    max(K_E3 e3, floor) is at least SEPARATION times below e2, the error of the 3-term scheme
    with one lo term dropped, both in the normalised max-norm and element-wise (error over the
    product scale sum |x| |w|).  A later loosening of K_E3 or the floor fails here."""
    torch.set_num_threads(max(1, os.cpu_count() or 8))
    cur, prev, metas, params, cfg = make_case(name)
    with torch.no_grad():
        m = metas[0]   # the arguments as oracle.dfm_backbone_forward builds them
        vol = O.build_dfm_cost(cur, prev, O.downsampled_depth(cfg), 1, 4,
                               torch.as_tensor(np.array([m['ori_cam2img']]), dtype=torch.float32),
                               torch.as_tensor(np.asarray(m['cur2prevs']), dtype=torch.float32),
                               m['ori_shape'][:2], m.get('flip', False), m['crop_offset'],
                               img_scale_factor=m['scale_factor'][0]).double()
        p = fp64_params(params, 'cpu')
        rows = []
        for mono in (False, True):
            out = {}
            for layer, x, w, mode, _ in tower_layers(vol, p, mono, out.__getitem__):
                if w is None:
                    out[layer] = x
                    continue
                ref = conv_planes(x, w, mode, 0, x.shape[2] * (2 if mode == 't' else 1)
                                  // (2 if mode == 's2' else 1))
                out[layer] = ref
                k = k_of(x.shape[1], mode)
                e3, e2 = emulate(x, w, mode, 0, ref.shape[2], ref)
                ys = emulated_outputs(x, w, mode, 0, ref.shape[2])
                _, el3, el2, elb = elementwise_errors(
                    ref, ref, *ys, product_scale(x, w, mode, 0, ref.shape[2]), k)
                rows.append((layer + ('_mono' if mono else ''), e3, e2, layer_bound(e3, k),
                             el3, el2, elb))
    print(f'\n{name}: layer | class | e3 | e2 | bound | e2 / bound || element-wise: '
          f'e3 | e2 | bound | e2 / bound')
    for layer, e3, e2, bound, el3, el2, elb in rows:
        print(f'  {layer:12s} {LAYER_CLASS[layer.replace("_mono", "")]:26s} {e3:.2e} {e2:.2e} '
              f'{bound:.2e} {e2 / bound:6.1f} || {el3:.2e} {el2:.2e} {elb:.2e} {el2 / elb:6.1f}')
    for layer, e3, e2, bound, el3, el2, elb in rows:
        assert e3 > 0 and e2 > 0 and el3 > 0, layer
        assert SEPARATION * bound <= e2, (layer, e3, e2, bound)
        assert SEPARATION * elb <= el2, (layer, 'element-wise', el3, el2, elb)


def test_slab_reference_matches_whole_volume():
    """conv_planes on slabs (halo, z padding, transposed phase) equals the whole-volume conv."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 8, 12, 5, 6, generator=g, dtype=torch.float64)
    w = torch.randn(4, 8, 3, 3, 3, generator=g, dtype=torch.float64)
    wt = torch.randn(8, 4, 3, 3, 3, generator=g, dtype=torch.float64)
    full = {'s1': F.conv3d(x, w, None, 1, 1), 's2': F.conv3d(x, w, None, 2, 1),
            't': F.conv_transpose3d(x, wt, None, 2, 1, 1)}
    for mode, y in full.items():
        for z0, z1 in ((0, 2), (2, 4), (0, y.shape[2]), (y.shape[2] - 2, y.shape[2])):
            got = conv_planes(x, wt if mode == 't' else w, mode, z0, z1)
            assert torch.allclose(got, y[:, :, z0:z1], rtol=0, atol=1e-12), (mode, z0, z1)


def test_z_expansion_maps():
    """The phase mapping of the shortened mono tower (simt_kernels.cuh ZExpand / zw_at)."""
    assert expand_index(68, 1, True)[:17] == list(range(17))
    assert expand_index(68, 1, True)[16:28] == [16, 17, 18, 19] * 3
    assert expand_index(68, 1, True)[-16:] == list(range(24, 40))
    assert expand_index(68, 2, True)[8:14] == [8, 9, 8, 9, 8, 9]
    assert expand_index(68, 4, True)[4:13] == [4] * 9
    assert computed_to_full(68, 2, True) == list(range(12)) + list(range(26, 34))
    assert expand_index(12, 1, False) == list(range(12))


# ---------------------------------------------------------------------------------------------
# z mapping of the shortened mono tower
# ---------------------------------------------------------------------------------------------
def shortened(d):
    return d >= 2 * Z_HEAD + 2 * Z_MID and os.environ.get('DFM_NO_ZSHORTEN') is None


def expand_index(d, s, short):
    """For every full plane at scale s, the computed plane that holds it."""
    df = d // s
    if not short:
        return list(range(df))
    head, period, shift = Z_HEAD // s, 4 // s, (d - 2 * Z_HEAD - Z_MID) // s
    return [z if z < head else z - shift if z >= df - head else head + (z - head) % period
            for z in range(df)]


def computed_to_full(d, s, short):
    """For every computed plane at scale s, the full plane it stands for."""
    if not short:
        return list(range(d // s))
    n, head, mid = (2 * Z_HEAD + Z_MID) // s, Z_HEAD // s, Z_MID // s
    shift = (d - 2 * Z_HEAD - Z_MID) // s
    return [j if j < head + mid else j + shift for j in range(n)]


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
CHANNELS = {'raw0': 32, 'cls3': 32, 'raw1': 32, 'c1': 64, 'c2': 64, 'c3': 64, 'c4': 64,
            'c5': 64, 'c6': 32, 'cur': 32, 'p0': 32, 'logit': 1}
LEVEL = {'raw0': 1, 'cls3': 1, 'raw1': 1, 'c1': 2, 'c2': 2, 'c3': 4, 'c4': 4, 'c5': 2, 'c6': 1,
         'cur': 1, 'p0': 1, 'logit': 1}
# kernel classes of the profile report (names without the shape) that compute a compared layer
TC_PREFIXES = ('conv_tc', 'cout1_logits', 'gate')
# every class the issue of this test names must be among them at the benchmarked shape
BENCH_CLASSES = ('conv_tc<32->32,s1,warp>', 'conv_tc<32->32,s1,src>', 'conv_tc_cl<32->64,s2,src>',
                 'conv_tc_ks<64->64,s2,src>', 'conv_tck<64->64,s1,src>', 'conv_tc<64->64,T,src>',
                 'conv_tc<64->32,T,src>', 'cout1_logits_tc<32->32,s1,src>', 'gate_tile4')
# the classes a case must have launched and compared
CASE_CLASSES = {'bench_384x1248_d112': BENCH_CLASSES,
                'gate_persistent_48x80_d120': ('gate_persistent',),
                'gate_v1_48x80_d148': ('gate_v1',)}


def _shell_mask(zidx, dz, h, w, tiles):
    """Boundary shell of the compared planes (indices zidx of the dz COMPUTED planes -- the
    kernels tile the computed volume -- of a [dz, h, w] grid): first / last plane, row and
    column, plus both sides of every tile seam (tiles = (tz, ty, tx), 0 = no seam there)."""
    shape = (len(zidx), h, w)
    m = torch.zeros(shape, dtype=torch.bool)
    for dim, (idx, n, t) in enumerate(zip((torch.tensor(zidx), torch.arange(h), torch.arange(w)),
                                          (dz, h, w), tiles)):
        sel = (idx == 0) | (idx == n - 1)
        if t:
            sel |= (idx % t == 0) | (idx % t == t - 1)
        view = [1, 1, 1]
        view[dim] = len(idx)
        m |= sel.view(view).expand(shape)
    return m


# (tz, ty, tx): conv_tc's M tile is 8 (x) by 16 (y) outputs (TC_BX, TC_BY in conv_tc.cuh);
# logits_tc's is 14 (x) by 6 (y) outputs and 16 planes (LT_OX, LT_OY, LT_ZC in logits_tc.cuh)
SHELL_TILES = {'raw0': (0, 16, 8), 'c1': (0, 16, 8), 'logit': (16, 6, 14)}


def _class_of(report, layer, mono, level_shape):
    """Kernel class that produced `layer` in this forward, from the profile report."""
    cin, cout, mode = {'raw0': (32, 32, 's1'), 'raw1': (32, 32, 's1'), 'c1': (32, 64, 's2'),
                       'c2': (64, 64, 's1'), 'c3': (64, 64, 's2'), 'c4': (64, 64, 's1'),
                       'c5': (64, 64, 'T'), 'c6': (64, 32, 'T'), 'p0': (32, 32, 's1'),
                       'logit': (32, 32, 's1')}[layer]
    suffix = '@' + 'x'.join(str(v) for v in level_shape)
    found = []
    for k in report:
        kind, _, rest = k.partition('<')
        if not k.endswith(suffix) or not rest.startswith(f'{cin}->{cout},{mode}'):
            continue
        if layer == 'logit' and 'cout1' not in kind and kind != 'conv_simt':
            continue
        if layer != 'logit' and 'cout1' in kind:
            continue
        if (layer == 'raw0') != (',warp>' in k):
            continue
        found.append(k.split('@')[0])
    return sorted(set(found))


def run_gpu_case(name):
    from depth_from_motion_b200 import capi, modules
    from tests.util import rel_err
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = 'cuda'
    cur, prev, metas, params, cfg = make_case(name)
    d = CASES[name]['d']
    ho, wo = CASES[name]['h'] // 4, CASES[name]['w'] // 4
    m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg, conv_impl='auto').cuda().eval()
    m.load_state_dict(params, strict=True)
    m.downsampled_depth = O.downsampled_depth(cfg)
    with torch.no_grad():
        m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))     # builds the handle and weights
        capi.sync_check()
        capi.profile_report()
        capi.profile_enable(True)
        try:
            cost, _, _ = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
            capi.sync_check()
            report = capi.profile_report()
        finally:
            capi.profile_enable(False)
        # dres0's input is the fp64 referee's volume, not the GPU's own warp: a defect shared
        # by the standalone op and the fused loaders cannot cancel out of the dres0 check
        g = PS.Geom.from_meta(metas[0])
        depths = O.downsampled_depth(cfg)
        cur_d, prev_d = cur.cuda().double(), prev.cuda().double()
        vol = PS.referee(cur_d, prev_d, depths, g)
        warp_b = PS.warp_input_bound(prev_d, vol[:, 32:], PS.sample_points(g, depths, ho, wo, dev),
                                     32)
        del cur_d, prev_d
    p = fp64_params(params, dev)
    short = shortened(d)
    slabs = slabs_of(name)
    rows, failures, checked = [], [], set()

    def gpu(layer, mono):
        """GPU tensor of a layer as computed: [1, C, Dc, H, W] fp64, Dc = computed planes."""
        s = LEVEL[layer]
        dc = 3 if layer == 'cls3' else ((2 * Z_HEAD + Z_MID) if (mono and short) else d) // s
        t = m.debug_tensor(layer + ('_mono' if mono else ''),
                           (dc, ho // s, wo // s, CHANNELS[layer]))
        return t.permute(3, 0, 1, 2)[None].double()

    def full(layer, mono):
        """The GPU tensor expanded to full depth (the reference consumes these)."""
        if layer == 'raw0' and mono:   # z-class compressed: first / interior / last plane
            return gpu('cls3', True)[:, :, [0] + [1] * (d - 2) + [2]]
        s = LEVEL[layer]
        return gpu(layer, mono)[:, :, expand_index(d, s, mono and short)]

    def compare(label, got, ref, k, e3e2, cls, shell=None, tol=None):
        """k = None: an fp32 element-wise stage (no products to split), held to tol.
        shell = (mask, y3, y2x, y2w, scale): element-wise check of the masked elements."""
        e = rel_err(got, ref)
        line = dict(case=name, layer=label, cls=cls, err=e)
        if k is not None:
            e3, e2 = e3e2
            bound = layer_bound(e3, k)
            line.update(e3=e3, e2=e2, bound=bound)
            if shell is not None:
                mask, *arrays = shell
                eg, el3, el2, elb = elementwise_errors(
                    got[..., mask], ref[..., mask], *(a[..., mask] for a in arrays), k)
                line.update(shell=eg, shell_bound=elb, shell_e2=el2)
                if eg > elb:
                    failures.append((label, 'shell element', eg, elb))
                if SEPARATION * elb > el2:
                    failures.append((label, 'shell separation', elb, el2))
            if e > bound:
                failures.append((label, e, bound))
            if SEPARATION * bound > e2:
                failures.append((label, 'separation', bound, e2))
        else:
            line['bound'] = tol
            if e > tol:
                failures.append((label, e, tol))
        rows.append(line)

    for mono in (False, True):
        tw = 'mono' if mono else 'stereo'
        sfx = '_mono' if mono else ''
        # the cur-frame half's z-class response: a z-invariant input on 3 planes gives the
        # first / interior / last plane of the full volume
        wcls = p[f'dres0{sfx}.conv.weight'][:, :32]
        xcls = vol[:, :32, :1].expand(-1, -1, 3, -1, -1)
        ref = conv_planes(xcls, wcls, 's1', 0, 3)
        classes = _class_of(report, 'raw0', mono, (5, ho, wo))
        checked.update(classes)
        compare(f'{tw}.cls3', gpu('cls3', mono), ref, k_of(32, 's1'),
                emulate(xcls, wcls, 's1', 0, 3, ref), ' | '.join(classes))
        c2f = {s: computed_to_full(d, s, mono and short) for s in (1, 2, 4)}
        for layer, x, w, mode, s in tower_layers(vol, p, mono, lambda n: full(n, mono)):
            if mono and layer == 'raw0':
                continue   # held as cls3_mono, checked above
            got_all = gpu(layer, mono)
            if layer == 'raw0':
                # the loader's warp error, bounded per input element (tests/plane_sweep_check.py):
                # each output may differ from the conv of the referee's volume by sum |w| times it
                got_all = got_all.clone()
                for z0, z1 in slabs:
                    ref = conv_planes(x, w, mode, z0, z1)
                    slack = conv_planes(warp_b, w.abs(), mode, z0, z1)
                    dv = got_all[:, :, z0:z1] - ref
                    got_all[:, :, z0:z1] = ref + dv.sign() * (dv.abs() - slack).clamp_min(0)
            el = layer in SHELL_TILES   # element-wise shell check
            gl, rl, e3s, e2s, zl, arrays = [], [], [], [], [], []
            for z0, z1 in slabs:
                z0s, z1s = z0 // s, z1 // s
                sel = [j for j, zf in enumerate(c2f[s]) if z0s <= zf < z1s]
                if not sel:
                    continue
                if w is None:
                    ref = x[:, :, z0s:z1s]
                else:
                    ref = conv_planes(x, w, mode, z0s, z1s)
                    e3, e2 = emulate(x, w, mode, z0s, z1s, ref)
                    e3s.append(e3)
                    e2s.append(e2)
                local = [c2f[s][j] - z0s for j in sel]
                if el:
                    arrays.append([a[:, :, local] for a in
                                   emulated_outputs(x, w, mode, z0s, z1s) +
                                   (product_scale(x, w, mode, z0s, z1s),)])
                gl.append(got_all[:, :, sel])
                rl.append(ref[:, :, local])
                zl += sel
            got, ref = torch.cat(gl, 2), torch.cat(rl, 2)
            if w is None:
                compare(f'{tw}.{layer}', got, ref, None, None, 'materialize', tol=1e-5)
                continue
            shell = None
            if el:
                shell = (_shell_mask(zl, len(c2f[s]), ho // s, wo // s, SHELL_TILES[layer]),) + \
                    tuple(torch.cat(a, 2) for a in zip(*arrays))
            dsz = (len(c2f[s]), ho // s, wo // s)
            classes = _class_of(report, layer, mono, dsz)
            checked.update(classes)
            compare(f'{tw}.{layer}', got, ref, k_of(x.shape[1], mode),
                    (max(e3s), min(e2s)), ' | '.join(classes), shell)
    # the mono / stereo gate on the GPU's own logits
    lg = gpu('logit', False)
    lm = full('logit', True)
    ref = gate(lg, lm, p['aggregate_cost.weight'])
    gate_classes = [k for k in report if k.startswith('gate')]
    checked.update(gate_classes)
    compare('gate', cost.double(), ref, None, None, ' | '.join(gate_classes), tol=1e-5)
    print(f'\n{name} (slabs {slabs}) kernel classes launched: {sorted(report)}')
    print('case | layer | kernel | GPU err | bound | e3 | e2 | err/e3 || shell element-wise: '
          'GPU | bound | e2')
    nan = float('nan')
    for r in rows:
        print(f"{r['case']} | {r['layer']} | {r['cls']} | {r['err']:.2e} | {r['bound']:.2e} | "
              f"{r.get('e3', nan):.2e} | {r.get('e2', nan):.2e} | "
              f"{r['err'] / r.get('e3', nan):.2f} || {r.get('shell', nan):.2e} | "
              f"{r.get('shell_bound', nan):.2e} | {r.get('shell_e2', nan):.2e}")
    print('CLASSES', ' '.join(sorted(report)))
    # every kernel class this forward launched for a compared layer was compared
    launched = {k.split('@')[0] for k in report if k.startswith(TC_PREFIXES)}
    if launched - checked:
        failures.append(('kernel classes launched but not compared', sorted(launched - checked)))
    return report, failures, checked


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_layers_vs_fp64(name):
    _, failures, checked = run_gpu_case(name)
    assert not failures, failures
    missing = [c for c in CASE_CLASSES.get(name, ()) if c not in checked]
    assert not missing, (missing, sorted(checked))


@pytest.mark.gpu
def test_layers_unshortened_mono_tower(monkeypatch):
    """DFM_NO_ZSHORTEN is read on every forward: the same layer check on the full-depth mono
    tower at a depth that is otherwise shortened."""
    monkeypatch.setenv('DFM_NO_ZSHORTEN', '1')
    _, failures, _ = run_gpu_case('aug_64x112_d68')
    assert not failures, failures


@pytest.mark.gpu
def test_debug_hook_refuses_unwritten_tensor():
    """On the z-class path dres0_mono's output lives in cls3_mono only: reading raw0_mono must
    fail instead of returning stale memory."""
    from depth_from_motion_b200 import modules
    cur, prev, metas, params, cfg = make_case('ragged_48x80_d12')
    m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg, conv_impl='auto').cuda().eval()
    m.load_state_dict(params, strict=True)
    with torch.no_grad():
        m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
    with pytest.raises(RuntimeError, match='not written'):
        m.debug_tensor('raw0_mono', (12, 12, 20, 32))
    assert m.debug_tensor('cls3_mono', (3, 12, 20, 32)).abs().max() > 0


# ---------------------------------------------------------------------------------------------
# A/B switch arms: the alternate kernels compute the same function
# ---------------------------------------------------------------------------------------------
AB_ARMS = [
    # (env, case, a class the arm must launch, a default-path class it must not launch).  The
    # default path launches the "avoid" class at that case, so each arm demonstrably switched.
    # the K-outer kernel is the default for conv2 / conv4 only where D-windows x tiles fill the
    # SMs: at 64 x 112 it never runs, so this arm runs at the shipped 320 x 1280, D = 72 shape
    ({'DFM_NO_NTK': '1'}, 'kitti_320x1280_d72', 'conv_tc<64->64,s1,src>@36x40x160', 'conv_tck'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('arm', AB_ARMS, ids=lambda a: ','.join(f'{k}={v}' for k, v in a[0].items()))
def test_ab_arm_layers(arm):
    """Each switch is fixed by the first call in a process, so each arm runs the per-layer
    test of its case in its own interpreter, against the same bounds."""
    env_add, case, want, avoid = arm
    env = dict(os.environ, **env_add)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-s',
                        '-m', 'gpu', '-p', 'no:cacheprovider', '-k',
                        f'test_layers_vs_fp64 and {case}'],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    print(out[-6000:])
    assert r.returncode == 0, out[-6000:]
    classes = [ln for ln in out.splitlines() if ln.startswith('CLASSES')]
    assert classes, out[-2000:]
    assert want in classes[0], classes[0]
    assert avoid not in classes[0], classes[0]


@pytest.mark.gpu
@pytest.mark.parametrize('wo,factor,tag', [(20, 4, 'depth_head'), (19, 3, 'depth_head_px1')],
                         ids=['20-4', '19-3'])
def test_depth_head_vs_oracle(wo, factor, tag):
    """dfm_depth_head_forward against oracle.depth_head_forward in fp64, at the default x4
    upsampling (four pixels per thread) and at an output width (19 x 3 = 57) that is not a
    multiple of 4, which takes the one-pixel-per-thread kernel."""
    from depth_from_motion_b200 import capi, modules
    from tests.util import rel_err
    d, ho = 12, 12
    g = torch.Generator().manual_seed(7)
    cost = torch.randn(1, 1, d, ho, wo, generator=g) * 3
    cfg = dict(num_bins=factor * d, depth_min=2, depth_max=59.6, downsample_factor=factor)
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2, max_depth=59.6),
        with_convs=False, num_views=1, depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = O.depth_samples(cfg)
    head.downsample_factor = factor
    cost = cost.cuda()
    capi.profile_enable(True)
    capi.profile_report()
    try:
        vol, sm, preds = head(cost)
        torch.cuda.synchronize()
        report = capi.profile_report()
    finally:
        capi.profile_enable(False)
    assert [k for k in report if k.startswith('depth_head')] == [tag], report
    rvol, rsm, rpreds = O.depth_head_forward(cost.cpu().double(), O.depth_samples(cfg).double(),
                                             factor)
    assert rel_err(vol, rvol) < 1e-5
    assert rel_err(sm, rsm) < 1e-5
    assert rel_err(preds, rpreds) < 1e-5
