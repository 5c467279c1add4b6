"""The stride-2 hourglass conv1 (32->64) on cluster-shared bricks.

By default the two output-channel groups of this conv run as one thread-block cluster whose CTAs
share every input brick through distributed shared memory (conv_tc.cuh, ``conv_tc_kernel``'s
CL).  DFM_S2_KSLICE=1, read whenever weights are set, selects the input-channel slices with
partial outputs in global memory instead.  The cluster route is checked here

* against fp64 with the per-layer bounds of ``tests/layer_check.py``, and against the K-slice
  route, through ``dfm_op_conv3d`` at the benchmarked shapes, at ragged tile remainders and on
  grids with fewer work units than SMs;
* inside the backbone, where the stereo tower's conv1 takes it (the mono tower's conv1 keeps
  the TMA-fed slices): against the K-slice route, on conv1 and conv3 of both towers and on the
  backbone outputs.  The per-layer fp64 test of the backbone (test_backbone_layers.py) checks
  both routes' classes at the benchmarked shape.
"""
import copy

import pytest
import torch

from tests import layer_check as LC

# (Di, Hi, Wi) of the 32-channel stride-2 input; Cout = 64
SHAPES = {
    # the stereo tower of the benchmarked KITTI step (D = 112, 384 x 1248 features)
    'bench': (112, 96, 312),
    # ragged 8 x 16 tiles: Ho = 19 = 16 + 3, Wo = 13 = 8 + 5 / Ho = 17, Wo = 21 = 16 + 5
    'ragged': (10, 38, 26),
    'ragged2': (6, 34, 42),
    # one tile column, 2 / 1 output planes: far fewer work units than clusters
    'few_units': (4, 16, 16),
    'one_unit': (2, 18, 14),
}
CLASS = {'cluster': 'conv_tc_cl', 'kslice': 'conv_tc_ks'}


def _conv(x, w, route, monkeypatch):
    from depth_from_motion_b200 import capi, modules
    if route == 'kslice':
        monkeypatch.setenv('DFM_S2_KSLICE', '1')
    else:
        monkeypatch.delenv('DFM_S2_KSLICE', raising=False)
    capi.profile_enable(True)
    capi.profile_report()
    y = modules.conv3d(x, w, stride=(2, 2, 2), padding=(1, 1, 1))
    torch.cuda.synchronize()
    report = capi.profile_report()
    capi.profile_enable(False)
    return y, sorted(k.split('@')[0] for k in report if k.startswith('conv'))


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(SHAPES))
def test_s2_conv_vs_fp64_and_kslice(name, monkeypatch):
    cin, (di, hi, wi) = 32, SHAPES[name]
    g = torch.Generator().manual_seed(list(SHAPES).index(name))
    x = torch.randn(1, cin, di, hi, wi, generator=g).cuda()
    w = (torch.randn(64, cin, 3, 3, 3, generator=g) / (27 * cin) ** 0.5).cuda()
    got = {}
    for route in ('cluster', 'kslice'):
        y, classes = _conv(x, w, route, monkeypatch)
        assert classes == [f'{CLASS[route]}<{cin}->64,s2,src>'], classes
        got[route] = y.double()
    xd, wd = x.double(), w.double()
    ref = LC.conv_planes(xd, wd, stride=2)
    e3, e2 = LC.emulate(xd, wd, ref, stride=2)
    bound = LC.layer_bound(e3, LC.k_of(cin))
    scale = float(ref.abs().max())
    err = float((got['cluster'] - ref).abs().max()) / scale
    print(f'{name}: err {err:.2e} bound {bound:.2e} e3 {e3:.2e} e2 {e2:.2e}')
    assert bound * LC.SEPARATION <= e2, (bound, e2)
    assert err <= bound, (err, bound)
    # the two routes differ only in the fp32 summation order of the same bf16 products
    diff = float((got['cluster'] - got['kslice']).abs().max()) / scale
    assert diff <= 1e-5, diff


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['aug_64x112_d68', 'bench_384x1248_d112'])
def test_backbone_routes_agree(case, monkeypatch):
    """conv1 / conv3 of the stereo and the z-shortened mono tower, and the backbone outputs,
    with the stereo conv1 on both routes from the same inputs."""
    from depth_from_motion_b200 import capi, modules
    from tests.test_backbone_layers import CASES, Z_HEAD, Z_MID, make_case
    cur, prev, metas, params, cfg = make_case(case)
    c = CASES[case]
    d, ho, wo = c['d'], c['h'] // 4, c['w'] // 4
    dm = 2 * Z_HEAD + Z_MID if d >= 2 * Z_HEAD + 2 * Z_MID else d   # computed mono planes
    shapes = {'c1': (d // 2, ho // 2, wo // 2, 64), 'c3': (d // 4, ho // 4, wo // 4, 64),
              'c1_mono': (dm // 2, ho // 2, wo // 2, 64), 'c3_mono': (dm // 4, ho // 4, wo // 4, 64)}
    got = {}
    for route in ('kslice', 'cluster'):
        if route == 'kslice':
            monkeypatch.setenv('DFM_S2_KSLICE', '1')
        else:
            monkeypatch.delenv('DFM_S2_KSLICE', raising=False)
        m = modules.DfMBackbone(in_channels=32, depth_cfg=cfg).cuda().eval()
        m.load_state_dict(params, strict=True)
        capi.profile_enable(True)
        capi.profile_report()
        with torch.no_grad():
            outs = m(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        torch.cuda.synchronize()
        report = capi.profile_report()
        capi.profile_enable(False)
        # the stereo conv1 (the K-slice route feeds it by TMA)
        stereo_c1 = f'@{d // 2}x{ho // 2}x{wo // 2}'
        assert any(k.startswith(f'{CLASS[route]}<32->64,s2,') and k.endswith(stereo_c1)
                   for k in report), report
        got[route] = dict(zip(('cost', 'stereo', 'mono'), (o.double() for o in outs)))
        got[route].update({n: m.debug_tensor(n, s).double() for n, s in shapes.items()})
        m.release()
    for n, ref in got['kslice'].items():
        diff = float((got['cluster'][n] - ref).abs().max()) / float(ref.abs().max())
        print(f'{case} {n}: cluster vs K-slice {diff:.2e}')
        assert diff <= 1e-5, (n, diff)
