"""The whole detectors against an fp64 reference detector built without the CUDA mirrors
(``tests/detector_reference.py``): same uint8 images, same state_dict, metas rebuilt from the
raw inputs.

CPU: the state_dict maps onto the restatements with every key read exactly once; the metas of
``prepare_kitti`` / ``prepare_waymo`` (pixel kernel stubbed) equal the rebuilt ones field by
field; the box comparator on hand-made cases at ``score_thr``, at ``nms_thr`` and at a dir-logit
tie; and, at small shapes, every join mistake of ``DEFECTS`` moves the head outputs by at least
``SEPARATION`` times the bound the GPU tests hold the head outputs to.

GPU (full size): ``DfM.simple_test`` (KITTI, B = 1 and a B = 2 batch of a 375 x 1242 and a
370 x 1224 pair) and ``MultiViewDfM.simple_test`` (camsync T = 1; 10-sweep T = 2 at B = 1 and
B = 2) against the fp64 reference at every stage join and on the final boxes.
"""
import copy
import gc
import math
import time

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import checkpoint, image_prep, modules
from depth_from_motion_b200 import synthetic as syn
from tests import box_post_oracle as BP
from tests import detector_reference as R
from tests.layer_check import SEPARATION
from tests.test_detector import CAMSYNC, CONFIGS, KITTI, SWEEPS10, build, random_state
from tests.util import rel_err

HEAD_BOUND = 1e-3          # north star: head outputs within 1e-3 (normalised max-norm)
# every join before the head is held to the same bar; at the shipped shapes they measure
# 1e-5 to 1e-4 on an H100 80GB HBM3 (700 W), the table the GPU tests print
JOIN_BOUND = 1e-3
# a kept box whose two direction logits are this close to a tie: the flip rule is live there
DIR_NEAR = 0.1


def kitti_images(seed, hw):
    """A smooth uint8 BGR pair, the previous frame shifted 3 px, as test_detector builds it."""
    rng = np.random.RandomState(seed)
    cur = (127 + 100 * np.tanh(syn.smooth_field(rng, 3, hw[0], hw[1], cell=16)[0].numpy()))
    cur = cur.astype(np.uint8).transpose(1, 2, 0).copy()
    return cur, np.roll(cur, 3, axis=1)


def waymo_images(seed, n, hw, cell=16):
    rng = np.random.RandomState(seed)
    return [(127 + 100 * np.tanh(syn.smooth_field(rng, 3, hw[0], hw[1], cell=cell)[0].numpy()))
            .astype(np.uint8).transpose(1, 2, 0).copy() for _ in range(n)]


def waymo_lidar2img(hw, num_frames):
    """syn.waymo_lidar2img's rig (focal length for a 1248-wide image) for raw images hw."""
    s = hw[1] / 1248.0
    return np.diag([s, s, 1, 1]) @ syn.waymo_lidar2img(num_frames)


# ---------------------------------------------------------------------------------------------
# small configs for the CPU tier: the shipped models on smaller grids
# ---------------------------------------------------------------------------------------------
def small_kitti():
    m = copy.deepcopy(CONFIGS[KITTI])
    m['voxel_cfg'] = dict(m['voxel_cfg'], point_cloud_range=[2, -6.4, -3, 14.8, 6.4, 1])
    for r in m['bbox_head_3d']['anchor_generator']['ranges']:
        r[0], r[1], r[3], r[4] = 2, -6.4, 14.8, 6.4
    return m


def small_waymo(name):
    m = copy.deepcopy(CONFIGS[name])
    m['anchor_generator']['ranges'] = [[0.0, -8.0, -2, 16.0, 8.0, 4]]   # in front of the rig
    for r in m['bbox_head_3d']['anchor_generator']['ranges']:
        r[0], r[1], r[3], r[4] = 0.0, -8.0, 16.0, 8.0
    return m


SMALL_KITTI = dict(hw=(275, 520), crop_size=(256, 512))   # SPP pools 64: f4 >= 64 x 128
SMALL_WAYMO = dict(hw=(100, 150), img_scale=(96, 64), num_views=2)


def _state(name, seed):
    det = build(name)
    state = random_state(det, seed)
    checkpoint.load_detector(state, det)
    return det, state


# ---------------------------------------------------------------------------------------------
# CPU: parameters
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,stages', [(KITTI, R.KITTI_STAGES), (SWEEPS10, R.WAYMO_STAGES),
                                         (CAMSYNC, R.WAYMO_STAGES)])
def test_state_dict_maps_onto_the_restatements(name, stages):
    det, state = _state(name, 3)
    params = R.split_state(det.state_dict(), stages)
    assert sum(len(p) for p in params.values()) == \
        sum(1 for k in state if not k.endswith('num_batches_tracked'))
    with pytest.raises(KeyError, match='onto 0'):
        R.split_state({**state, 'stray.weight': torch.zeros(1)}, stages)
    with pytest.raises(KeyError, match='onto 2'):
        R.split_state(state, stages + (('backbone.conv1', 'twice'),))


def _kitti_small_run(defect=None, seed=5):
    det, _ = _state(KITTI, seed)
    params = R.split_state(det.state_dict(), R.KITTI_STAGES)
    cur, prev = kitti_images(seed, SMALL_KITTI['hw'])
    meta = R.kitti_metas(SMALL_KITTI['hw'], syn.KITTI_P2, syn.KITTI_CUR2PREV[2:3],
                         crop_size=SMALL_KITTI['crop_size'])
    with torch.no_grad():
        out = R.kitti_forward(params, small_kitti(), cur, prev, meta,
                              crop_size=SMALL_KITTI['crop_size'], defect=defect)
    return out, params


def _waymo_small_run(name, defect=None, seed=6):
    det, _ = _state(name, seed)
    params = R.split_state(det.state_dict(), R.WAYMO_STAGES)
    t = 2 if name == SWEEPS10 else 1
    nv, hw = SMALL_WAYMO['num_views'], SMALL_WAYMO['hw']
    views = waymo_images(seed, nv * t, hw, cell=8)
    l2i = syn.waymo_lidar2img(t, nv)
    l2i = np.diag([hw[1] / 1248.0, hw[1] / 1248.0, 1, 1]) @ l2i
    meta = R.waymo_metas(hw, l2i, nv, t - 1, img_scale=SMALL_WAYMO['img_scale'])
    with torch.no_grad():
        out = R.waymo_forward(params, small_waymo(name), views, meta,
                              img_scale=SMALL_WAYMO['img_scale'], defect=defect)
    return out, params


def test_every_parameter_is_read_kitti():
    _, params = _kitti_small_run()
    assert R.unread(params) == []


@pytest.mark.parametrize('name', [SWEEPS10, CAMSYNC])
def test_every_parameter_is_read_waymo(name):
    _, params = _waymo_small_run(name)
    assert R.unread(params) == []


# ---------------------------------------------------------------------------------------------
# CPU: metas
# ---------------------------------------------------------------------------------------------
def _cpu_prep(monkeypatch):
    """prepare_kitti / prepare_waymo with the pixel kernel stubbed: their metas, on the CPU."""
    monkeypatch.setattr(image_prep, '_to_device_views',
                        lambda views, device: torch.stack([torch.as_tensor(v) for v in views]))

    def fake(src, mode, out_hw, crop_xy=(0, 0), size_divisor=32, *a, **k):
        return torch.zeros((src.shape[0], 3, -(-out_hw[0] // size_divisor) * size_divisor,
                            -(-out_hw[1] // size_divisor) * size_divisor))
    monkeypatch.setattr(image_prep, 'image_prep', fake)


def _plain(x):
    if isinstance(x, torch.Tensor):
        x = x.numpy()
    if isinstance(x, np.ndarray):
        x = x.tolist()
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x.item() if isinstance(x, np.generic) else x


def assert_same_metas(lib, ref, keys):
    """Field by field; float fields to fp32 precision (the library keeps fp32 copies of the
    matrices, which the reference converts to fp32 where it reads them)."""
    for k in keys:
        a, b = _plain(lib[k]), _plain(ref[k])
        if np.asarray(b).dtype.kind == 'f':
            np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64),
                                       rtol=2.0 ** -23, atol=1e-6, err_msg=k)
        else:
            assert a == b, (k, a, b)


KITTI_META_KEYS = ('ori_cam2img', 'cam2img', 'cur2prevs', 'ori_shape', 'img_shape', 'pad_shape',
                   'crop_offset', 'flip', 'scale_factor')
WAYMO_META_KEYS = ('ori_lidar2img', 'scale_factor', 'ori_shape', 'img_shape', 'pad_shape',
                   'num_views', 'num_ref_frames')


@pytest.mark.parametrize('hw,crop', [((375, 1242), (320, 1280)), ((370, 1224), (320, 1280)),
                                     ((275, 520), (256, 512)), ((300, 1300), (320, 1280))])
def test_kitti_metas_match_prepare_kitti(hw, crop, monkeypatch):
    _cpu_prep(monkeypatch)
    cur, prev = kitti_images(1, hw)
    c2p = syn.KITTI_CUR2PREV[1:2]
    _, (lib,) = image_prep.prepare_kitti(cur, [prev], syn.KITTI_P2, c2p, device='cpu',
                                          crop_size=crop)
    ref = R.kitti_metas(hw, syn.KITTI_P2, c2p, crop_size=crop)
    assert_same_metas(lib, ref, KITTI_META_KEYS)
    # and a meta that is wrong is told apart
    bad = dict(ref, crop_offset=[ref['crop_offset'][0], ref['crop_offset'][1] + 1])
    with pytest.raises(AssertionError):
        assert_same_metas(lib, bad, KITTI_META_KEYS)


@pytest.mark.parametrize('hw,t', [((1280, 1920), 1), ((886, 1920), 2), ((100, 150), 2)])
def test_waymo_metas_match_prepare_waymo(hw, t, monkeypatch):
    _cpu_prep(monkeypatch)
    views = [np.zeros(hw + (3,), np.uint8)] * (5 * t)
    l2i = waymo_lidar2img(hw, t)
    scale = (96, 64) if hw == (100, 150) else (1248, 832)
    _, (lib,) = image_prep.prepare_waymo(views, l2i, num_ref_frames=t - 1, device='cpu',
                                          img_scale=scale)
    ref = R.waymo_metas(hw, l2i, 5, t - 1, img_scale=scale)
    assert_same_metas(lib, ref, WAYMO_META_KEYS)
    assert tuple(ref['input_shape']) == tuple(lib['pad_shape'][0][:2])


# ---------------------------------------------------------------------------------------------
# CPU: the box comparator on hand-made cases
# ---------------------------------------------------------------------------------------------
def _hand_model():
    m = copy.deepcopy(CONFIGS[KITTI])
    gen = m['bbox_head_3d']['anchor_generator']
    for r in gen['ranges']:
        r[0], r[1], r[3], r[4] = 0.0, 0.0, 9.0, 1.0
    m['test_cfg'] = dict(m['test_cfg'], nms_pre=4096, max_num=500)
    return m


def _hand_heads():
    """A 2 x 10 BEV grid, 6 anchors per cell, every score far below score_thr except the
    boxes each case places."""
    cls = torch.full((18, 2, 10), -8.0, dtype=torch.float64)
    box = torch.zeros((42, 2, 10), dtype=torch.float64)
    dirc = torch.zeros((12, 2, 10), dtype=torch.float64)
    dirc[0::2] = 1.0                     # direction 0 clear everywhere
    return cls, box, dirc


def _got(model, cls, box, dirc):
    r = R.boxes(model, cls.float().double(), box.float().double(), dirc.float().double())
    return r['boxes'].float(), r['scores'].float(), r['labels']


def _logit(p):
    return math.log(p / (1 - p))



def test_box_comparator_hand_cases():
    m = _hand_model()
    thr, nms_thr = m['test_cfg']['score_thr'], m['test_cfg']['nms_thr']
    e = 1e-3
    cls, box, dirc = _hand_heads()
    # anchor (cell y0 x1, class 0 size, rot 0) = channel 0: a clear box
    cls[0, 0, 1] = 2.0
    # a box right at score_thr: channel 0 at cell (0, 8)
    cls[0, 0, 8] = _logit(thr) + 0.5 * e
    # two class-0 boxes two cells apart, stretched along x so that their BEV IoU is nms_thr
    cls[0, 1, 3], cls[0, 1, 5] = 1.0, 0.9
    # dir-logit tie at the clear box
    dirc[0, 0, 1] = dirc[1, 0, 1] = 0.3
    table = R.anchors(m['bbox_head_3d']['anchor_generator'], 2, 10).double()
    a3, a5 = (1 * 10 + 3) * 6, (1 * 10 + 5) * 6
    # w (box dim 3, along x at yaw 0): two boxes `gap` apart overlap by IoU (w - gap) / (w + gap)
    gap = float(table[a5, 0] - table[a3, 0])

    def width_code(a, iou):
        return math.log(gap * (1 + iou) / (1 - iou) / float(table[a, 3]))
    for a, ch in ((a3, (1, 3)), (a5, (1, 5))):
        box[3, ch[0], ch[1]] = width_code(a, nms_thr - 0.3 * R.IOU_TOL)
    ref = R.boxes(m, cls, box, dirc)
    assert ref['boxes'].shape[0] == 4, ref['scores']
    iou = float(BP.rotated_iou(BP.nms_box(ref['boxes'][1:2]), BP.nms_box(ref['boxes'][2:3])))
    assert abs(iou - (nms_thr - 0.3 * R.IOU_TOL)) < 1e-9, iou

    def run(c, b, d):
        return R.compare_boxes(_got(m, c, b, d), m, cls, box, dirc, e, e, e)
    # within the bounds: the library drops the threshold box, suppresses the pair's second box
    # and flips the tied direction
    c2, b2, d2 = cls.clone(), box.clone(), dirc.clone()
    c2[0, 0, 8] -= e
    # the second box of the pair widened so that the pair's IoU is just above nms_thr:
    # w1 + w2 = 2 gap (1 + iou) / (1 - iou)
    t = nms_thr + 0.3 * R.IOU_TOL
    w1 = float(torch.exp(box[3, 1, 3])) * float(table[a3, 3])
    b2[3, 1, 5] = math.log((2 * gap * (1 + t) / (1 - t) - w1) / float(table[a5, 3]))
    d2[1, 0, 1] += 0.5 * e
    r = run(c2, b2, d2)
    print('hand cases', r)
    assert r['failures'] == [] and r['matched'] == 2 and r['exempt'] == 2
    # a clear box missing, a score beyond the bound, a flip without a tie: each one fails
    c3 = cls.clone()
    c3[0, 0, 1] = -8.0
    assert any('kept by the reference only' in f for f in run(c3, box, dirc)['failures'])
    c4 = cls.clone()
    c4[0, 1, 3] += 20 * e
    assert run(c4, box, dirc)['failures']
    d5 = dirc.clone()
    d5[0, 1, 3], d5[1, 1, 3] = 0.0, 1.0
    assert any('direction flipped' in f for f in run(cls, box, d5)['failures'])
    # every library box emitted twice: each second copy fails
    g = _got(m, cls, box, dirc)
    twice = tuple(torch.cat([x, x]) for x in g)
    r = R.compare_boxes(twice, m, cls, box, dirc, e, e, e)
    assert sum('both anchor' in f for f in r['failures']) == g[0].shape[0] == 4
    # the first box of the pair (direction label clear) with its yaw just past limit_period's
    # boundary in the reference and just before it in the library: pi apart, one label
    b6 = box.clone()
    off = m['bbox_head_3d']['dir_offset']
    b6[6, 1, 3] = off + math.pi - float(table[a3, 6]) + 0.3 * e
    g6 = b6.clone()
    g6[6, 1, 3] -= 0.6 * e
    got6 = _got(m, cls, g6, dirc)
    ref6 = R.boxes(m, cls, b6, dirc)
    assert abs(abs(float(got6[0][1, 6] - ref6['boxes'][1, 6])) - math.pi) < 2 * e
    r = R.compare_boxes(got6, m, cls, b6, dirc, e, e, e)
    assert r['failures'] == [] and r['matched'] == 4, r


# ---------------------------------------------------------------------------------------------
# CPU: every join mistake moves the head outputs far beyond the bound
# ---------------------------------------------------------------------------------------------
def _head_move(a, b):
    return max(rel_err(a[k], b[k]) for k in ('cls', 'box', 'dir'))


def test_kitti_join_defects_are_seen():
    good, _ = _kitti_small_run()
    assert float((good['volume'] != 0).double().mean()) > 0.2
    for defect in R.KITTI_DEFECTS:
        bad, _ = _kitti_small_run(defect)
        move = _head_move(bad, good)
        print('kitti defect', defect, 'head move', move, 'ratio', move / HEAD_BOUND)
        assert move >= SEPARATION * HEAD_BOUND, defect


@pytest.mark.parametrize('name', [SWEEPS10, CAMSYNC])
def test_waymo_join_defects_are_seen(name):
    good, _ = _waymo_small_run(name)
    assert float((good['volume'] != 0).double().mean()) > 0.2
    for defect in R.WAYMO_DEFECTS:
        bad, _ = _waymo_small_run(name, defect)
        move = _head_move(bad, good)
        print('waymo defect', name, defect, 'head move', move, 'ratio', move / HEAD_BOUND)
        assert move >= SEPARATION * HEAD_BOUND, defect


# ---------------------------------------------------------------------------------------------
# GPU: the shipped detectors at full size
# ---------------------------------------------------------------------------------------------
# Random init leaves every class logit within about +-2 of 0, every score far above the
# configs' score_thr (0.1 KITTI, 0.001 Waymo), so the threshold, the nms_pre cut and NMS among
# near-equal scores would never be exercised.  The final class conv is scaled and its bias
# moved to logit(score_thr) so that scores spread across the threshold.  Likewise the random
# direction classifier gives the high-scoring Waymo boxes dir-logit margins of 0.3 to 3 (its
# biases alone differ by 0.1 to 0.3 within a pair), so no kept box would sit near a tie: each
# pair's biases are made equal and its weights scaled by DIR_GAIN.
CLS_GAIN = 3.0
DIR_GAIN = 0.1


def _cuda_detector(name, seed):
    from tests.test_detector import _free
    _free()
    det = build(name)
    state = random_state(det, seed)
    thr = CONFIGS[name]['test_cfg']['score_thr']
    state['bbox_head_3d.conv_cls.weight'] = state['bbox_head_3d.conv_cls.weight'] * CLS_GAIN
    state['bbox_head_3d.conv_cls.bias'] = state['bbox_head_3d.conv_cls.bias'] + _logit(thr)
    state['bbox_head_3d.conv_dir_cls.weight'] *= DIR_GAIN
    dir_bias = state['bbox_head_3d.conv_dir_cls.bias'].view(-1, 2)
    state['bbox_head_3d.conv_dir_cls.bias'] = dir_bias[:, :1].expand(-1, 2).reshape(-1).clone()
    checkpoint.load_detector(state, det)
    return det.cuda().eval()


def _gpu_kitti_joins(det, img, metas):
    """DfM's mirrors one by one for one sample (test_detector.kitti_by_hand), keeping every
    join."""
    metas = copy.deepcopy(metas)
    cur_imgs, prev_imgs = img[:, 0], img[:, 1]
    cur_feats = [cur_imgs] + list(det.backbone(cur_imgs))
    prev_feats = [prev_imgs] + list(det.backbone(prev_imgs))
    cur_stereo, cur_sem = det.neck(cur_feats)
    prev_stereo, _ = det.neck(prev_feats)
    for m in metas:
        m['cur2prevs'] = torch.tensor(np.asarray(m['cur2prevs']), dtype=img.dtype)
    costs, stereo, _ = det.backbone_stereo(cur_stereo, prev_stereo, metas)
    lg = modules.CostLogits(costs, depth_samples=det.depth_head.depth_samples)
    volume = det.feature_transformation(stereo, lg, metas, cur_sem)
    _, cv, nz, ny, nx = volume.shape
    _, bev = det.backbone_3d(volume.view(-1, cv * nz, ny, nx))
    cls, box, dirc = det.bbox_head_3d([bev])
    return dict(img=cur_imgs, img_feat=cur_feats[-1], stereo_in=cur_stereo, sem=cur_sem,
                cost=costs, stereo=stereo, depth_preds=lg.depth_preds, volume=volume, bev=bev,
                cls=cls[0], box=box[0], dir=dirc[0])


def _gpu_waymo_joins(det, img, metas):
    metas = copy.deepcopy(metas)
    nv, t = metas[0]['num_views'], metas[0]['num_ref_frames'] + 1
    feats = det.neck(det.backbone(img.reshape(-1, *img.shape[2:])))[0]
    meta = dict(metas[0], input_shape=img.shape[-2:])
    volume = modules.multiview_lift(feats, meta, list(det.n_voxels), list(det.voxel_range), nv,
                                    t, det.temporal_aggregate)[None]
    bev = det.neck_3d(volume)[0]
    cls, box, dirc = det.bbox_head_3d([bev])
    return dict(img=img[0], feat=feats, volume=volume, bev=bev, cls=cls[0], box=box[0],
                dir=dirc[0])


def _compare(what, got, ref, model, result):
    """Every join within its bound, then the boxes.  Prints the whole table before asserting."""
    errs = {}
    for k in ref:
        if k in got:
            assert got[k].numel() == ref[k].numel(), (k, got[k].shape, ref[k].shape)
            errs[k] = rel_err(got[k].reshape(ref[k].shape), ref[k])
    for k, e in errs.items():
        bound = HEAD_BOUND if k in ('cls', 'box', 'dir') else JOIN_BOUND
        print(f'{what} join {k:12s} rel err {e:.3e} bound {bound:.0e}')
    vol = ref['volume']
    nonzero = float((vol != 0).double().mean())
    thr = model['test_cfg']['score_thr']
    scores = ref['cls'][0].double().sigmoid()
    above = float((scores > thr).double().mean())
    e = {k: HEAD_BOUND * float(ref[k][0].abs().max()) for k in ('cls', 'box', 'dir')}
    r = R.compare_boxes(result, model, ref['cls'][0], ref['box'][0], ref['dir'][0],
                        e['cls'], e['box'], e['dir'])
    close = sum(m < DIR_NEAR for m in r['dir_margins'])
    tied = sum(m <= 2 * e['dir'] for m in r['dir_margins'])
    print(f'{what}: voxels non-zero {nonzero:.3f}, scores above score_thr {above:.3f}, '
          f'kept boxes with dir logits within {DIR_NEAR} {close} (within the bound {tied}), '
          f'boxes {r["total"]} matched {r["matched"]} exempt {r["exempt"]}')
    for f in r['failures'][:20]:
        print(what, 'box failure:', f)
    assert nonzero > 0.2
    assert 0.01 < above < 0.9
    assert close > 0
    assert r['total'] >= 20
    for k, err in errs.items():
        assert err <= (HEAD_BOUND if k in ('cls', 'box', 'dir') else JOIN_BOUND), (what, k, err)
    assert r['failures'] == [], r['failures'][:5]
    assert r['exempt'] <= R.MAX_EXEMPT * max(r['total'], 1)


def _ref_kitti(det, name, cur, prev, c2p):
    params = R.split_state(det.state_dict(), R.KITTI_STAGES, device='cuda')
    meta = R.kitti_metas(cur.shape[:2], syn.KITTI_P2, c2p)
    out = R.kitti_forward(params, CONFIGS[name], cur, prev, meta)
    assert R.unread(params) == []
    return out, meta


def _result(r):
    return r['boxes_3d'], r['scores_3d'], r['labels_3d']


@pytest.mark.gpu
@pytest.mark.parametrize('batch', [1, 2])
def test_kitti_detector_vs_fp64_reference(batch):
    """B = 1: a 375 x 1242 pair.  B = 2: that pair and a 370 x 1224 one in one batch, each
    sample bitwise equal to its own B = 1 call and against the reference."""
    from tests.test_detector import _free, _same
    t0 = time.perf_counter()
    det = _cuda_detector(KITTI, 41)
    try:
        samples = [(kitti_images(42, (375, 1242)), syn.KITTI_CUR2PREV[2:3]),
                   (kitti_images(43, (370, 1224)), syn.KITTI_CUR2PREV[1:2])][:batch]
        imgs, metas = [], []
        for (cur, prev), c2p in samples:
            img, m = image_prep.prepare_kitti(cur, [prev], syn.KITTI_P2, c2p)
            assert img.shape == (1, 2, 3, 320, 1248)
            assert_same_metas(m[0], R.kitti_metas(cur.shape[:2], syn.KITTI_P2, c2p),
                              KITTI_META_KEYS)
            imgs.append(img)
            metas += m
        with torch.no_grad():
            one = [det.simple_test(imgs[b], copy.deepcopy(metas[b:b + 1]))[0]
                   for b in range(batch)]
            if batch > 1:
                both = det.simple_test(torch.cat(imgs), copy.deepcopy(metas))
                _same(both, one, 'kitti B=2')
            for b, ((cur, prev), c2p) in enumerate(samples):
                got = _gpu_kitti_joins(det, imgs[b], metas[b:b + 1])
                ref, _ = _ref_kitti(det, KITTI, cur, prev, c2p)
                _compare(f'kitti B={batch} sample {b}', got, ref, CONFIGS[KITTI], _result(one[b]))
                del got, ref
                gc.collect()
                torch.cuda.empty_cache()
    finally:
        _free(det)
    print(f'kitti B={batch} wall time {time.perf_counter() - t0:.1f} s')


@pytest.mark.gpu
@pytest.mark.parametrize('name,num_frames,batch', [(CAMSYNC, 1, 1), (SWEEPS10, 2, 1),
                                                         (SWEEPS10, 2, 2)])
def test_waymo_detector_vs_fp64_reference(name, num_frames, batch):
    from tests.test_detector import _free, _same
    t0 = time.perf_counter()
    det = _cuda_detector(name, 51)
    hw = (1280, 1920)
    l2i = waymo_lidar2img(hw, num_frames)
    try:
        imgs, metas, raw = [], [], []
        for b in range(batch):
            views = waymo_images(52 + b, 5 * num_frames, hw)
            img, m = image_prep.prepare_waymo(views, l2i, num_ref_frames=num_frames - 1)
            assert img.shape == (1, 5 * num_frames, 3, 832, 1248)
            ref_meta = R.waymo_metas(hw, l2i, 5, num_frames - 1)
            assert_same_metas(m[0], ref_meta, WAYMO_META_KEYS)
            imgs.append(img)
            metas += m
            raw.append((views, ref_meta))
        with torch.no_grad():
            one = [det.simple_test(imgs[b], copy.deepcopy(metas[b:b + 1]))[0]
                   for b in range(batch)]
            if batch > 1:
                both = det.simple_test(torch.cat(imgs), copy.deepcopy(metas))
                _same(both, one, 'waymo B=2')
            for b in range(batch):
                got = _gpu_waymo_joins(det, imgs[b], metas[b:b + 1])
                params = R.split_state(det.state_dict(), R.WAYMO_STAGES, device='cuda')
                ref = R.waymo_forward(params, CONFIGS[name], *raw[b])
                assert R.unread(params) == []
                _compare(f'{name} T={num_frames} sample {b}', got, ref, CONFIGS[name],
                         _result(one[b]))
                del got, ref, params
                gc.collect()
                torch.cuda.empty_cache()
    finally:
        _free(det)
    print(f'{name} T={num_frames} B={batch} wall time {time.perf_counter() - t0:.1f} s')
