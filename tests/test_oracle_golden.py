"""CPU tests: the oracle restatement against (1) the reference's own golden vectors
for this path (SURVEY.md section 8c) and (2) fixtures produced by the unmodified
reference sources (tests/golden/make_golden.py)."""
import math
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import synthetic as syn
from oracle import dfm_oracle as O
from tests.util import GOLDEN, KITTI_CASES, assert_close, load_kitti_case


def test_points_img2cam_kat():
    # reference tests/test_utils/test_utils.py:186-193
    points = torch.tensor([[0.5764, 0.9109, 0.7576], [0.6656, 0.5498, 0.9813]])
    cam2img = torch.tensor([[700., 0., 450., 0.], [0., 700., 200., 0.],
                            [0., 0., 1., 0.]])
    expected = torch.tensor([[-0.4864, -0.2155, 0.7576],
                             [-0.6299, -0.2796, 0.9813]])
    assert torch.allclose(O.points_img2cam(points, cam2img), expected, atol=1e-3)


def test_points_cam2img_kat():
    # reference tests/test_utils/test_box3d.py:1653-1680
    torch.manual_seed(0)
    points = torch.rand([5, 3])
    proj_mat = torch.rand([4, 4])
    expected = torch.tensor([[0.5832, 0.6496], [0.6146, 0.7910],
                             [0.6994, 0.7782], [0.5623, 0.6303],
                             [0.4359, 0.6532]])
    assert torch.allclose(O.points_cam2img(points, proj_mat), expected, 1e-3)
    expected_d = torch.tensor([[0.5832, 0.6496, 1.7577], [0.6146, 0.7910, 1.5477],
                               [0.6994, 0.7782, 2.0091], [0.5623, 0.6303, 1.8739],
                               [0.4359, 0.6532, 1.2056]])
    assert torch.allclose(O.points_cam2img(points, proj_mat, with_depth=True),
                          expected_d, 1e-3)


def test_point_sample_kat():
    # reference tests/test_models/test_fusion/test_point_fusion.py:13-41 (the
    # no-3D-augmentation half; PointFusion.sample_single -> point_sample with
    # scale 1, crop 0, no flip, bilinear, align_corners=True)
    lidar2img = torch.tensor(
        [[6.0294e+02, -7.0791e+02, -1.2275e+01, -1.7094e+02],
         [1.7678e+02, 8.8088e+00, -7.0794e+02, -1.0257e+02],
         [9.9998e-01, -1.5283e-03, -5.2907e-03, -3.2757e-01],
         [0.0000e+00, 0.0000e+00, 0.0000e+00, 1.0000e+00]])
    img_feat = torch.arange(370 * 1224)[None, ...].view(
        370, 1224)[None, None, ...].float() / (370 * 1224)
    pts = torch.tensor([[8.356, -4.312, -0.445], [11.777, -6.724, -0.564],
                        [6.453, 2.53, -1.612], [6.227, -3.839, -0.563]])
    out = O.point_sample(img_feat, pts, lidar2img, pts.new_tensor([1., 1.]),
                         0, False, (370, 1224), (370, 1224), aligned=True)
    expected = torch.tensor([0.5560822, 0.5476625, 0.9687978, 0.6241757])
    assert torch.allclose(expected, out.squeeze(), 1e-4)


@pytest.mark.parametrize('name', sorted(KITTI_CASES))
def test_backbone_matches_reference_fixture(name):
    cur, prev, metas, params, cfg, gold = load_kitti_case(name)
    spec = KITTI_CASES[name]
    with torch.no_grad():
        vol = O.build_dfm_cost(
            cur, prev, O.downsampled_depth(cfg), 1, 4,
            torch.as_tensor(np.array([metas[0]['ori_cam2img']]),
                            dtype=torch.float32), metas[0]['cur2prevs'],
            metas[0]['ori_shape'][:2], spec[4], metas[0]['crop_offset'],
            img_scale_factor=spec[6])
        cost, stereo, mono = O.dfm_backbone_forward(params, cur, prev, metas, cfg)
        _, sm, preds = O.depth_head_forward(cost, O.depth_samples(cfg))
    # same ATen ops in the same order; CPU kernels of another instruction set round
    # differently (FMA contraction in grid_sample / conv): up to ~2e-4 absolute on values of a
    # few units, so the absolute term scales with the tensor (|d| <= 1e-4 |b| + 5e-5 max|b|)
    for got, key in ((vol, 'volume'), (cost, 'cost'), (stereo, 'stereo'),
                     (mono, 'mono'), (preds, 'depth_preds')):
        ref = torch.from_numpy(gold[key])
        assert got.shape == ref.shape, key
        assert_close(got, ref, key, rtol=1e-4, atol_frac=5e-5)
    assert torch.allclose(sm[0, 0, :, ::8, ::8],
                          torch.from_numpy(gold['softmax_slice']), atol=1e-6)


def test_generated_inputs_match_stored_inputs():
    # fixture inputs regenerate bit-identically from their seed
    for name, spec in KITTI_CASES.items():
        seed, h, w, d = spec[:4]
        cur, prev, _, _ = syn.make_kitti_pair(seed, h, w, d)
        gold = np.load(os.path.join(GOLDEN, name + '.npz'))
        assert np.array_equal(cur.numpy(), gold['cur'])
        assert np.array_equal(prev.numpy(), gold['prev'])


@pytest.mark.parametrize('name', ['neck_dfm', 'neck_imvoxel'])
def test_neck_matches_reference_fixture(name):
    from depth_from_motion_b200 import modules
    gold = np.load(os.path.join(GOLDEN, name + '.npz'))
    rng = np.random.RandomState(21)
    dfm = modules.DfMNeck(64, 256, num_frames=2)
    imv = modules.OutdoorImVoxelNeck(64, 256)
    # make_golden draws the DfMNeck parameters first, then its input, then the
    # OutdoorImVoxelNeck parameters: replay the same stream
    sd_dfm = syn.make_neck_params(rng, dfm.state_dict())
    x_dfm = rng.standard_normal((1, 128, 6, 5, 12)).astype(np.float32)
    sd_imv = syn.make_neck_params(rng, imv.state_dict())
    x = torch.from_numpy(gold['x'])
    if name == 'neck_dfm':
        assert np.array_equal(x_dfm, gold['x'])
        with torch.no_grad():
            y = O.dfm_neck_forward(sd_dfm, x, 64)[0]
    else:
        with torch.no_grad():
            y = O.imvoxel_neck_forward(sd_imv, x)[0]
    assert torch.allclose(y, torch.from_numpy(gold['y']), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('name', ['neck_dfm_mt', 'neck_imvoxel_mt'])
def test_neck_multitile_fixture(name):
    """The multi-tile neck fixtures (37 x 21 x 12 voxels = 3 x 3 tiles of the CUDA kernel,
    ragged edges): inputs regenerate from the seed (checksums stored), the oracle restatement
    reproduces the verbatim reference output."""
    from depth_from_motion_b200 import modules
    from tests.util import make_neck_mt_case
    gold = np.load(os.path.join(GOLDEN, name + '.npz'))
    rng, x = make_neck_mt_case(name)
    # (a double sum: its last bit depends on the host's summation kernel)
    assert math.isclose(float(x.double().sum()), float(gold['x_sum']), rel_tol=1e-14)
    assert math.isclose(float(x.double().abs().sum()), float(gold['x_abs']), rel_tol=1e-14)
    mod = (modules.DfMNeck(64, 256, num_frames=2) if name == 'neck_dfm_mt'
           else modules.OutdoorImVoxelNeck(64, 256))
    sd = syn.make_neck_params(rng, mod.state_dict())
    with torch.no_grad():
        y = (O.dfm_neck_forward(sd, x, 64) if name == 'neck_dfm_mt'
             else O.imvoxel_neck_forward(sd, x))[0]
    ref = torch.from_numpy(gold['y'])
    assert y.shape == ref.shape == (1, 256, 21, 37)
    assert torch.allclose(y, ref, rtol=1e-4, atol=1e-4)


def test_depth_tables():
    cfg = syn.depth_cfg_for(72)
    d = O.downsampled_depth(cfg)
    assert d.shape == (72,) and abs(float(d[0]) - (2 + 0.5 * 4 * 0.2)) < 1e-5
    s = O.depth_samples(cfg)
    assert s.shape == (288,) and abs(float(s[-1]) - (59.6 - 0.1)) < 1e-4


def test_frustum_to_voxel_matches_reference_fixture():
    """SURVEY.md section 8(f) row 1: oracle restatement (DepthHead -> FrustumToVoxel)
    against the verbatim reference run stored in tests/golden/frustum.npz."""
    from tests.util import load_frustum_case
    c, gold = load_frustum_case()
    cfg = c['depth_cfg']
    _, sm, _ = O.depth_head_forward(c['cost'], O.depth_samples(cfg), 4)
    assert torch.equal(sm, torch.from_numpy(gold['softmax']))
    out = O.frustum_to_voxel_forward(c['params'], c['stereo'], sm, c['metas'], c['sem'],
                                     c['coordinates_3d'], cfg)
    ref = torch.from_numpy(gold['out'])
    assert out.shape == ref.shape == (1, 32, 2, 20, 24)
    assert_close(out, ref, 'frustum', rtol=1e-5, atol_frac=1e-6)
    # the grid of the shipped config (detectors/dfm.py:174-211)
    full = O.frustum_coordinates_3d(dict(point_cloud_range=syn.KITTI_POINT_CLOUD_RANGE,
                                         voxel_size=syn.KITTI_VOXEL_SIZE))
    assert tuple(full.shape) == (20, 304, 288, 3)
    assert torch.equal(full, syn.frustum_coordinates(syn.KITTI_POINT_CLOUD_RANGE,
                                                     (288, 304, 20)))


def voxel_sample_args(flip):
    """Inputs of the voxel_sample comparison (also used by tests/golden/make_reference_io.py)."""
    g = torch.Generator().manual_seed(3)
    vox = torch.randn(1, 6, 20, 16, 8, generator=g)
    vrange, vsize = [0.0, -8.0, -2.0, 20.0, 8.0, 2.0], [1.0, 1.0, 0.5]
    depths = torch.linspace(2.0, 18.0, 16)
    # lidar -> image: camera looks along +x
    k = torch.tensor([[40., 0, 32, 0], [0, 40., 16, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    l2c = torch.tensor([[0., -1, 0, 0], [0, 0, -1, 0.3], [1, 0, 0, 0.1], [0, 0, 0, 1]])
    proj = k @ l2c
    return (vox, vrange, vsize, depths, proj, 4, torch.tensor([1.02, 0.98]),
            torch.tensor([1.0, 2.0]), flip, (32, 64), (30, 62))


def _reference_io(key):
    return torch.from_numpy(np.load(os.path.join(GOLDEN, 'reference_io.npz'))[key])


@pytest.mark.parametrize('flip,aligned', [(False, True), (True, True), (False, False)])
def test_voxel_sample_matches_reference_source(flip, aligned):
    """SURVEY.md row a8 (oracle only): the restatement against the output of the reference
    function executed verbatim (point_fusion.py:324-410), stored in reference_io.npz."""
    a = _reference_io(f'voxel_sample_{int(flip)}_{int(aligned)}')
    b = O.voxel_sample(*voxel_sample_args(flip), aligned=aligned)
    assert a.shape == b.shape == (1, 6, 4, 8, 16)
    assert_close(b, a, 'voxel_sample', rtol=1e-5, atol_frac=2e-6)   # (stored on another host)
    assert float(a.abs().sum()) > 0


def test_bev_stage_matches_reference_fixture():
    """SURVEY.md section 8(f) row 3: oracle restatement of BEVHourglass + LIGAAnchor3DHead
    (class scores, 3-D box regressions, direction logits) against the verbatim reference run."""
    gold = np.load(os.path.join(GOLDEN, 'bev_stage.npz'))
    c = syn.make_bev_case(**syn.BEV_CASE)
    assert math.isclose(float(c['volume'].double().sum()), float(gold['x_sum']), rel_tol=1e-14)
    v = c['volume']
    with torch.no_grad():
        prehg, bev = O.bev_hourglass_forward(c['bev'], v.reshape(1, -1, v.shape[3], v.shape[4]))
        outs = O.dfm_bev_stage(c['bev'], c['head'], v)
    for got, key in ((prehg, 'prehg'), (bev, 'bev'), (outs[0], 'cls_score'),
                     (outs[1], 'bbox_pred'), (outs[2], 'dir_cls_preds')):
        ref = torch.from_numpy(gold[key])
        assert got.shape == ref.shape, key
        assert torch.allclose(got, ref, rtol=1e-4, atol=1e-5), key
    assert outs[0].shape[1] == 18 and outs[1].shape[1] == 42 and outs[2].shape[1] == 12


def test_bev_stage_oracle_equals_reference_source():
    """Against the output of the reference classes executed in place (reference_io.npz); the
    tolerance covers CPU kernels that round differently on another host."""
    c = syn.make_bev_case(seed=5, nz=5, ny=12, nx=16)
    with torch.no_grad():
        got = O.dfm_bev_stage(c['bev'], c['head'], c['volume'])
    assert len(got) == 3
    for i, a in enumerate(got):
        ref = _reference_io(f'bev_small_{i}')
        assert_close(a, ref, f'bev output {i}', rtol=1e-5, atol_frac=2e-6)


def test_spp_unet_lastconv_equals_reference_module():
    """SURVEY.md section 8(f) row 2: the oracle restatement of SPPUNetNeck.lastconv against the
    reference class executed in place (spp_unet_neck.py:60-75, :110), stored with its randomly
    initialised parameters in reference_io.npz."""
    gold = np.load(os.path.join(GOLDEN, 'reference_io.npz'))
    p = {k.split(':', 1)[1]: torch.from_numpy(gold[k]) for k in gold.files
         if k.startswith('lastconv_param:')}
    assert sorted(p) == ['lastconv.0.conv.weight', 'lastconv.0.gn.bias', 'lastconv.0.gn.weight',
                         'lastconv.1.weight']
    x = torch.randn(1, 32, 24, 40, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        assert_close(O.spp_unet_lastconv(p, x), torch.from_numpy(gold['lastconv_out']), 'lastconv',
                     rtol=1e-5, atol_frac=2e-6)
    # the mirror takes the same keys
    from depth_from_motion_b200 import modules
    modules.SPPUNetNeckTail().load_state_dict(p, strict=True)
