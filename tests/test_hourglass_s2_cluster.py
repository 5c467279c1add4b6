"""The stride-2 hourglass conv1 (32->64) on cluster-shared bricks.

The two output-channel groups of this conv run as one thread-block cluster whose CTAs share every
input brick through distributed shared memory (conv_tc.cuh, ``conv_tc_kernel``'s CL).  This route
is checked here against fp64 with the per-layer bounds of ``tests/layer_check.py``, through
``dfm_op_conv3d`` at the benchmarked shape, at ragged tile remainders and on grids with fewer work
units than SMs.  Inside the backbone both towers' conv1 take it; the per-layer fp64 test of the
backbone (test_backbone_layers.py) checks conv1 and conv3 of both towers.
"""
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


def _conv(x, w):
    from depth_from_motion_b200 import capi, modules
    capi.profile_enable(True)
    capi.profile_report()
    y = modules.conv3d(x, w, stride=(2, 2, 2), padding=(1, 1, 1))
    torch.cuda.synchronize()
    report = capi.profile_report()
    capi.profile_enable(False)
    return y, sorted(k.split('@')[0] for k in report if k.startswith('conv'))


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(SHAPES))
def test_s2_conv_vs_fp64(name):
    cin, (di, hi, wi) = 32, SHAPES[name]
    g = torch.Generator().manual_seed(list(SHAPES).index(name))
    x = torch.randn(1, cin, di, hi, wi, generator=g).cuda()
    w = (torch.randn(64, cin, 3, 3, 3, generator=g) / (27 * cin) ** 0.5).cuda()
    y, classes = _conv(x, w)
    assert classes == [f'conv_tc_cl<{cin}->64,s2,src>'], classes
    xd, wd = x.double(), w.double()
    ref = LC.conv_planes(xd, wd, stride=2)
    e3, e2 = LC.emulate(xd, wd, ref, stride=2)
    bound = LC.layer_bound(e3, LC.k_of(cin))
    scale = float(ref.abs().max())
    err = float((y.double() - ref).abs().max()) / scale
    print(f'{name}: err {err:.2e} bound {bound:.2e} e3 {e3:.2e} e2 {e2:.2e}')
    assert bound * LC.SEPARATION <= e2, (bound, e2)
    assert err <= bound, (err, bound)
