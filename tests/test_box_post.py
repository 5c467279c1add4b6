"""get_bboxes of both anchor heads (dense_heads/anchor3d_head.py:407-547, box3d_nms.py) on CUDA
(``dfm_box_post_*``, ``modules.{LIGAAnchor3DHead,Anchor3DHead}.get_bboxes``).

CPU: the torch restatement ``tests/box_post_oracle.py`` reproduces ``tests/golden/box_post.npz``
(written by the reference's own functions) bit for bit; the module's anchor tables equal the
reference generators'; the nms_rotated stand-in on hand-worked pairs; the descriptor ABI.
GPU: synthetic head outputs at the shipped grids and the real regressions of both all-CUDA
chains, fed to the library and to the restatement on the same GPU tensors."""
import ctypes
import hashlib
import math
import os
import subprocess
import shutil

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import synthetic as syn
from tests import box_post_oracle as BP
from tests.util import GOLDEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-5


def _golden():
    return np.load(os.path.join(GOLDEN, 'box_post.npz'))


def _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset, num_classes=3):
    with torch.no_grad():
        return BP.get_bboxes_single(cls, box, dirc, anchors, cfg, num_classes, sigmoid,
                                    dir_offset, 0.0)


# ---------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize('name', list(syn.BOX_POST_CASES))
def test_oracle_matches_reference_golden(name):
    generator, ny, nx, cfg, sigmoid, dir_offset, seed, kw = syn.BOX_POST_CASES[name]
    g = _golden()
    cls, box, dirc = syn.make_box_post_case(seed, ny, nx, **kw)
    assert sum(t.double().abs().sum().item() for t in (cls, box, dirc)) == \
        float(g[f'{name}.input_sum'])
    anchors = modules.grid_anchors(generator, ny, nx, 'cpu')
    assert torch.equal(anchors, torch.from_numpy(g[f'{name}.anchors']))
    r = _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset)
    assert torch.equal(r['boxes'], torch.from_numpy(g[f'{name}.boxes']))
    assert torch.equal(r['scores'], torch.from_numpy(g[f'{name}.scores']))
    assert torch.equal(r['labels'], torch.from_numpy(g[f'{name}.labels']))
    n_anchor = ny * nx * 6
    assert (r['topk'] is not None) == (n_anchor > cfg['nms_pre'])
    if name == 'kitti_max_num_empty_class':
        assert len(r['candidates'][2]) == 0 and len(r['boxes']) == cfg['max_num']
        assert sum(len(k) for k in r['keep']) > cfg['max_num']


@pytest.mark.parametrize('name,generator,ny,nx', [
    ('kitti', syn.KITTI_ANCHOR_GENERATOR, 304, 288), ('waymo', syn.WAYMO_ANCHOR_GENERATOR, 300, 220)])
def test_anchor_table_at_shipped_grid(name, generator, ny, nx):
    g = _golden()
    a = modules.grid_anchors(generator, ny, nx, 'cpu').contiguous()
    assert tuple(a.shape) == tuple(g[f'{name}_full.shape'])
    assert hashlib.sha256(a.numpy().tobytes()).hexdigest() == str(g[f'{name}_full.anchors_sha256'])


def _box(x, y, w, h, r):
    return torch.tensor([x, y, w, h, r], dtype=torch.float64)


def test_rotated_iou_hand_cases():
    """Identical boxes: 1.  Disjoint: 0.  A unit square at 45 degrees centred in a 2 x 2 square
    lies inside it: IoU = 1 / 4."""
    a = _box(3.0, -2.0, 4.0, 1.5, 0.7)
    assert float(BP.rotated_iou(a, a)) == pytest.approx(1.0, abs=1e-12)
    assert float(BP.rotated_iou(a, _box(30.0, 5.0, 4.0, 1.5, 0.7))) == 0.0
    assert float(BP.rotated_iou(_box(1, 1, 2, 2, 0.0), _box(1, 1, 1, 1, math.pi / 4))) == \
        pytest.approx(0.25, abs=1e-12)


def test_rotated_iou_corner_convention(monkeypatch):
    """Two 4 x 1 boxes at yaw pi/4, centres (0, 0) and (1, 1).  With mmcv's corners
    (centre + R(-yaw)(+-w/2, +-h/2)) the long axis runs along (1, -1)/sqrt 2: the centre offset
    (1, 1) is perpendicular to it at distance sqrt 2 > h = 1, so the boxes are disjoint, IoU 0,
    below nms_thr 0.25.  With R(+yaw) (LiDARInstance3DBoxes.corners) the long axis runs along
    the offset: overlap (4 - sqrt 2) x 1 = 2.586, union 8 - 2.586 = 5.414, IoU 0.4776 > 0.25."""
    a, b = _box(0, 0, 4, 1, math.pi / 4), _box(1, 1, 4, 1, math.pi / 4)
    assert BP.NMS_ROTATED_ROT_SIGN == -1.0
    assert float(BP.rotated_iou(a, b)) == 0.0
    monkeypatch.setattr(BP, 'NMS_ROTATED_ROT_SIGN', 1.0)
    s2 = math.sqrt(2)
    assert float(BP.rotated_iou(a, b)) == pytest.approx((4 - s2) / (4 + s2), abs=1e-12)


def test_kernel_states_the_same_convention():
    src = open(os.path.join(ROOT, 'depth_from_motion_b200', 'csrc', 'box_post_kernels.cuh')).read()
    assert 'constexpr float BP_ROT_SIGN = -1.f;' in src


@pytest.mark.skipif(shutil.which('gcc') is None, reason='no C compiler')
def test_box_post_desc_matches_the_c_header(tmp_path):
    cls = capi.BoxPostDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>',
             f'#include "{os.path.join(ROOT, "include", "dfm_b200.h")}"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(dfm_box_post_desc_t));']
    lines += [f'printf("{f} %zu\\n", offsetof(dfm_box_post_desc_t, {f}));' for f, _ in cls._fields_]
    lines += ['return 0;', '}']
    (tmp_path / 'abi.c').write_text('\n'.join(lines))
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-o', str(tmp_path / 'abi'),
                    str(tmp_path / 'abi.c')], check=True)
    got = dict(l.split() for l in subprocess.run([str(tmp_path / 'abi')], capture_output=True,
                                                 text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _kitti_head(**cfg):
    return modules.LIGAAnchor3DHead(
        num_classes=3, in_channels=64, feat_channels=64, norm_cfg=dict(type='GN', num_groups=32),
        anchor_generator=syn.KITTI_ANCHOR_GENERATOR, dir_offset=syn.KITTI_DIR_OFFSET,
        test_cfg=dict(syn.KITTI_TEST_CFG, **cfg))


def _waymo_head(sigmoid=True, **cfg):
    return modules.Anchor3DHead(
        num_classes=3, in_channels=256, anchor_generator=syn.WAYMO_ANCHOR_GENERATOR,
        dir_offset=syn.WAYMO_DIR_OFFSET, test_cfg=dict(syn.WAYMO_TEST_CFG, **cfg),
        loss_cls=dict(type='FocalLoss', use_sigmoid=sigmoid))


def test_unsupported_options_raise():
    cls, box, dirc = (t[None] for t in syn.make_box_post_case(1, 4, 4))
    with pytest.raises(NotImplementedError):
        _kitti_head(use_rotate_nms=False).get_bboxes([cls], [box], [dirc], [{}])
    with pytest.raises(NotImplementedError):
        _waymo_head().get_bboxes([cls], [box], None, [{}])
    with pytest.raises(NotImplementedError):
        _waymo_head().get_bboxes([cls], [box], [None], [{}])
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        _waymo_head().get_bboxes([cls], [box], [dirc], [{}])


# ---------------------------------------------------------------------------------- GPU

def _nms_validity(bev, cand, keep, thr):
    """fp64 IoU in processing order: a kept box overlaps no earlier kept box by more than
    thr + EPS; a suppressed one overlaps some earlier kept box by more than thr - EPS.  Returns
    the number of decisions within EPS of thr."""
    n = len(cand)
    if n == 0:
        return 0
    pos = {int(a): i for i, a in enumerate(cand.tolist())}
    kept = torch.zeros(n, dtype=torch.bool, device=bev.device)
    kept[[pos[int(a)] for a in keep.tolist()]] = True
    iou = BP.rotated_iou(bev[:, None], bev[kept][None])           # [n, kept]
    kidx = torch.nonzero(kept).flatten()
    earlier = kidx[None, :] < torch.arange(n, device=bev.device)[:, None]
    m = torch.where(earlier, iou, torch.full_like(iou, -1.0)).max(dim=1)[0]
    assert bool((m[kept] <= thr + EPS).all()), float(m[kept].max())
    assert bool((m[~kept] > thr - EPS).all()), float(m[~kept].min())
    return int(((m - thr).abs() <= EPS).sum())


def _check_against_oracle(head, cls, box, dirc, anchors, cfg, sigmoid, dir_offset, label):
    """One sample through head.get_bboxes and the oracle on the same GPU tensors."""
    (boxes, scores, labels), = head.get_bboxes([cls[None]], [box[None]], [dirc[None]], [{}])
    capi.sync_check()
    r = _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset)
    bp = head._box_post
    # top-k, tie-aware
    if r['topk'] is not None:
        got = bp.debug_tensor('topk_index')[0].long()
        ref = r['topk']
        ncol = 3 if sigmoid else 4
        sc = cls.permute(1, 2, 0).reshape(-1, ncol)
        sc = (sc.sigmoid() if sigmoid else sc.softmax(-1)[:, :-1]).max(1)[0]
        assert torch.equal(torch.sort(sc[got], descending=True)[0], sc[got]), 'not sorted'
        kth = sc[ref[-1]]
        diff_g = set(got.tolist()) - set(ref.tolist())
        diff_r = set(ref.tolist()) - set(got.tolist())
        assert all(float(sc[i]) == float(kth) for i in diff_g | diff_r), 'top-k differs off ties'
    # candidates and keeps per class
    ties_band = 0
    bev_all = None
    same_keep = True
    slot_anchor = r['topk'] if r['topk'] is not None else torch.arange(cls.shape[-1] *
                                                                       cls.shape[-2] * 6,
                                                                       device=cls.device)
    with torch.no_grad():
        dec = BP.decode(anchors[slot_anchor],
                        box.permute(1, 2, 0).reshape(-1, 7)[slot_anchor])
        bev_all = BP.nms_box(dec)
    slot_of = torch.full((anchors.shape[0],), -1, dtype=torch.long, device=cls.device)
    slot_of[slot_anchor] = torch.arange(len(slot_anchor), device=cls.device)
    for c in range(3):
        cand = bp.debug_tensor(f'cls{c}_candidates')[0].long()
        cand = cand[cand >= 0]
        keep = bp.debug_tensor(f'cls{c}_keep')[0].long()
        keep = keep[keep >= 0]
        assert set(cand.tolist()) == set(r['candidates'][c].tolist()), (label, c)
        band = _nms_validity(bev_all[slot_of[cand]], cand, keep, cfg['nms_thr'])
        ties_band += band
        if band == 0:
            assert torch.equal(keep, r['keep'][c]), (label, c)
        same_keep &= torch.equal(keep, r['keep'][c])
        print(label, 'class', c, 'candidates', len(cand), 'kept', len(keep), 'band', band)
    if same_keep:
        assert torch.equal(labels, r['labels'])
        assert torch.equal(scores, r['scores'])
        torch.testing.assert_close(boxes, r['boxes'], rtol=2.4e-7, atol=1e-6)
    return boxes, scores, labels, ties_band


@pytest.mark.gpu
@pytest.mark.parametrize('shape', ['kitti', 'waymo'])
def test_shipped_shape_vs_oracle(shape):
    if shape == 'kitti':
        ny, nx, head, gen = 304, 288, _kitti_head(), syn.KITTI_ANCHOR_GENERATOR
        cfg, dir_offset = syn.KITTI_TEST_CFG, syn.KITTI_DIR_OFFSET
    else:
        ny, nx, head, gen = 300, 220, _waymo_head(), syn.WAYMO_ANCHOR_GENERATOR
        cfg, dir_offset = syn.WAYMO_TEST_CFG, syn.WAYMO_DIR_OFFSET
    cls, box, dirc = (t.cuda() for t in syn.make_box_post_case(11, ny, nx))
    anchors = modules.grid_anchors(gen, ny, nx, 'cuda')
    l0, _ = capi.launch_counters()
    boxes, scores, labels, band = _check_against_oracle(head, cls, box, dirc, anchors, cfg, True,
                                                        dir_offset, shape)
    assert capi.launch_counters()[0] > l0
    assert 0 < len(boxes) <= cfg['max_num']
    print(shape, 'boxes', len(boxes), 'decisions within EPS of nms_thr', band)


@pytest.mark.gpu
def test_softmax_arm_vs_oracle():
    generator, ny, nx, cfg, sigmoid, dir_offset, seed, kw = syn.BOX_POST_CASES['waymo_softmax']
    cls, box, dirc = (t.cuda() for t in syn.make_box_post_case(seed, ny, nx, **kw))
    anchors = modules.grid_anchors(generator, ny, nx, 'cuda')
    head = _waymo_head(sigmoid=False, **{k: v for k, v in cfg.items()})
    # softmax: scores may differ from torch's by rounding; check the NMS and the set sizes
    (boxes, scores, labels), = head.get_bboxes([cls[None]], [box[None]], [dirc[None]], [{}])
    r = _oracle(cls, box, dirc, anchors, cfg, False, dir_offset)
    assert len(boxes) == len(r['boxes'])
    torch.testing.assert_close(scores, r['scores'], rtol=1e-6, atol=1e-7)


def _run(head, cls, box, dirc, metas):
    out = head.get_bboxes([cls], [box], [dirc], metas)
    capi.sync_check()
    return out


@pytest.mark.gpu
def test_repeatable_batched_and_empty():
    ny, nx = 300, 220
    cases = [syn.make_box_post_case(s, ny, nx) for s in (21, 22)]
    cls, box, dirc = (torch.stack([c[i] for c in cases]).cuda() for i in range(3))
    head = _waymo_head()
    a = _run(head, cls, box, dirc, [{}, {}])
    b = _run(head, cls, box, dirc, [{}, {}])
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    single = _waymo_head()
    for i in range(2):
        (bx, sc, lb), = _run(single, cls[i:i + 1], box[i:i + 1], dirc[i:i + 1], [{}])
        assert torch.equal(bx, a[i][0]) and torch.equal(sc, a[i][1]) and torch.equal(lb, a[i][2])
    # nothing passes score_thr
    (bx, sc, lb), = _run(_waymo_head(score_thr=0.9999), torch.full_like(cls[:1], -9.0), box[:1],
                         dirc[:1], [{}])
    assert bx.shape == (0, 7) and sc.shape == (0,) and lb.shape == (0,)


def _desc(**kw):
    d = dict(num_classes=3, num_anchors=6, ny=300, nx=220, batch=1, use_sigmoid=1, nms_pre=4096,
             max_num=500, score_thr=0.001, nms_thr=0.05, dir_offset=-0.7854,
             dir_limit_offset=0.0)
    d.update(kw)
    return capi.BoxPostDesc(*[d[f] for f, _ in capi.BoxPostDesc._fields_])


@pytest.mark.gpu
def test_c_api_canaries_and_errors():
    L = capi.lib()
    ny, nx = 300, 220
    anchors = modules.grid_anchors(syn.WAYMO_ANCHOR_GENERATOR, ny, nx, 'cpu').contiguous()
    hd = ctypes.c_void_p()
    for bad in (dict(nms_pre=0), dict(nms_pre=5000), dict(num_classes=0), dict(num_classes=17),
                dict(batch=0), dict(max_num=0), dict(use_sigmoid=2), dict(nms_thr=float('nan'))):
        assert L.dfm_box_post_create(ctypes.byref(_desc(**bad)), modules._ptr(anchors),
                                     ctypes.byref(hd)) == 1, bad
    assert L.dfm_box_post_create(ctypes.byref(_desc()), None, ctypes.byref(hd)) == 1
    capi.check(L.dfm_box_post_create(ctypes.byref(_desc(max_num=50)), modules._ptr(anchors),
                                     ctypes.byref(hd)), 'create')
    try:
        cls, box, dirc = (t[None].cuda() for t in syn.make_box_post_case(31, ny, nx))
        boxes = torch.full((1, 50, 7), 123.0, device='cuda')
        scores = torch.full((1, 50), 123.0, device='cuda')
        labels = torch.full((1, 50), 77, device='cuda', dtype=torch.int32)
        count = torch.full((1,), -1, device='cuda', dtype=torch.int32)
        p = modules._ptr
        s = modules._stream()
        assert L.dfm_box_post_forward(hd, p(cls), p(box), None, p(boxes), p(scores), p(labels),
                                      p(count), s) == 1
        out = torch.empty(4096, device='cuda', dtype=torch.int32)
        assert L.dfm_box_post_debug_tensor(hd, b'topk_index', p(out), 4096, s) == 3
        # a tiny max_num with many kept boxes: exactly max_num written
        capi.check(L.dfm_box_post_forward(hd, p(cls), p(box), p(dirc), p(boxes), p(scores),
                                          p(labels), p(count), s), 'forward')
        capi.sync_check()
        assert int(count[0]) == 50
        assert L.dfm_box_post_debug_tensor(hd, b'topk_index', p(out), 4095, s) == 1
        assert L.dfm_box_post_debug_tensor(hd, b'cls9_keep', p(out), 4096, s) == 1
        # a sample with few boxes: canaries past count stay
        boxes.fill_(123.0)
        scores.fill_(123.0)
        labels.fill_(77)
        cls2 = torch.full_like(cls, -9.0)
        cls2[0, 0, 100, 100] = 3.0
        capi.check(L.dfm_box_post_forward(hd, p(cls2), p(box), p(dirc), p(boxes), p(scores),
                                          p(labels), p(count), s), 'forward')
        capi.sync_check()
        k = int(count[0])
        assert 1 <= k < 50
        assert bool((boxes[0, k:] == 123.0).all()) and bool((scores[0, k:] == 123.0).all())
        assert bool((labels[0, k:] == 77).all())
    finally:
        L.dfm_box_post_destroy(hd)


@pytest.mark.gpu
def test_kitti_chain_end_to_end():
    """The real regressions of test_box_regression_parity_end_to_end's all-CUDA KITTI chain
    (DfMBackbone -> FrustumToVoxel -> BEVHourglass -> LIGAAnchor3DHead) through get_bboxes."""
    import copy

    from oracle import dfm_oracle as O
    from tests.test_gpu_parity import _backbone, _bev_modules, _frustum_module
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(23, h, w, d)
    cfg = syn.depth_cfg_for(d)
    fc = syn.make_frustum_case(24, h, w, d, (32, 28, 20))
    metas = copy.deepcopy(metas)
    metas[0]['cam2img'] = fc['metas'][0]['cam2img']
    bc = syn.make_bev_case(seed=25, nz=5, ny=28, nx=32)
    bb, fr = _backbone(params, cfg, 'auto'), _frustum_module(fc)
    bev, head = _bev_modules(bc)
    with torch.no_grad():
        cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        vol = fr(stereo, modules.CostLogits(cost, depth_samples=O.depth_samples(cfg)), metas,
                 fc['sem'].cuda())
        _, nz, ny, nx = vol.shape[1:]
        _, feat = bev(vol.view(1, -1, ny, nx))
        cls, box, dirc = head([feat])
    head.extra_cfg['anchor_generator'] = syn.KITTI_ANCHOR_GENERATOR
    head.extra_cfg['dir_offset'] = syn.KITTI_DIR_OFFSET
    cfg = dict(syn.KITTI_TEST_CFG, score_thr=0.3)
    head.test_cfg = cfg
    anchors = modules.grid_anchors(syn.KITTI_ANCHOR_GENERATOR, ny, nx, 'cuda')
    _check_against_oracle(head, cls[0][0], box[0][0], dirc[0][0], anchors, cfg, True,
                          syn.KITTI_DIR_OFFSET, 'kitti chain')


@pytest.mark.gpu
def test_waymo_chain_end_to_end():
    """lifting -> DfMNeck -> Anchor3DHead (the chain of test_waymo_box_regressions_end_to_end)
    through get_bboxes, two samples in one call checked one by one."""
    from tests.test_anchor3d_head import _cuda_head, load_fixture
    torch.backends.cudnn.allow_tf32 = False
    nv, t = 3, 2
    n_voxels, vrange = [20, 18, 12], [0.0, -9.0, -2.0, 20.0, 9.0, 4.0]
    rng = np.random.RandomState(61)
    mod = modules.DfMNeck(64, 256, num_frames=2)
    mod.load_state_dict(syn.make_neck_params(rng, mod.state_dict()), strict=True)
    mod = mod.cuda().eval()
    _, hp = load_fixture()
    head = _cuda_head(hp)

    class Host(modules.MultiViewDfMFeatureTransformation):
        pass
    host = Host()
    host.n_voxels, host.voxel_range = n_voxels, vrange
    host.temporal_aggregate, host.valid_sample, host.neck_3d = 'concat', True, mod
    feats, metas = [], []
    for b in range(2):
        f, m = syn.make_waymo_sample(70 + b, t, nv, feat_hw=(40, 64), input_hw=(160, 256),
                                     flip=bool(b), scale=1.0 + 0.02 * b, crop=(1.0 * b, 2.0 * b))
        k = np.array([[120., 0, 128, 0], [0, 120., 80, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        kfull = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        m['ori_lidar2img'] = np.array([k @ np.linalg.inv(kfull) @ x
                                       for x in syn.waymo_lidar2img(t, nv)])
        feats.append(f)
        metas.append(m)
    with torch.no_grad():
        bev = host.feature_transformation(torch.stack(feats).cuda(), metas, nv, t)[0]
        cls, box, dirc = head([bev])
    head.extra_cfg['anchor_generator'] = syn.WAYMO_ANCHOR_GENERATOR
    head.dir_offset = syn.WAYMO_DIR_OFFSET
    head.test_cfg = syn.WAYMO_TEST_CFG
    ny, nx = cls[0].shape[-2:]
    anchors = modules.grid_anchors(syn.WAYMO_ANCHOR_GENERATOR, ny, nx, 'cuda')
    both = head.get_bboxes(cls, box, dirc, [{}, {}])
    capi.sync_check()
    for b in range(2):
        got = _check_against_oracle(head, cls[0][b], box[0][b], dirc[0][b], anchors,
                                    syn.WAYMO_TEST_CFG, True, syn.WAYMO_DIR_OFFSET,
                                    f'waymo chain {b}')
        for u, v in zip(both[b], got[:3]):
            assert torch.equal(u, v)
