"""KITTI evaluation (depth_from_motion_b200.kitti_eval, csrc/kitti_eval_kernels.cuh) against
the golden of mmdet3d's evaluator (tests/golden/make_kitti_eval_golden.py) and against the
host restatement in oracle/kitti_eval_oracle.py."""
import ctypes
import json
import math
import os

import numpy as np
import pytest

from depth_from_motion_b200 import kitti_eval as ke
from oracle import kitti_eval_oracle as orc

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
CLASSES = ['Car', 'Pedestrian', 'Cyclist']


def load_golden():
    z = dict(np.load(os.path.join(GOLDEN, 'kitti_eval.npz')))
    with open(os.path.join(GOLDEN, 'kitti_eval.json')) as f:
        meta = json.load(f)

    def unpack(prefix, keys):
        off = z[f'{prefix}_off']
        return [{k: z[f'{prefix}_{k}'][off[i]:off[i + 1]] for k in keys}
                for i in range(len(off) - 1)]

    gts = unpack('gt', ('name', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y',
                        'occluded', 'truncated'))
    dts = unpack('dt', ('name', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y',
                        'score'))
    return z, meta, gts, dts


def golden_overlaps(z, gts, dts):
    """per metric, the list of per-frame [dt, gt] golden overlaps"""
    out = {}
    for m in range(3):
        flat, pos, frames = z[f'overlap{m}'], 0, []
        for g, d in zip(gts, dts):
            n = len(d['name']) * len(g['name'])
            frames.append(flat[pos:pos + n].reshape(len(d['name']), len(g['name'])))
            pos += n
        out[m] = frames
    return out


def anno(names, bbox, loc, dims, ry, alpha=None, score=None, occluded=None, truncated=None):
    n = len(names)
    a = dict(name=np.array(names, dtype='<U14'), bbox=np.array(bbox, np.float64).reshape(n, 4),
             location=np.array(loc, np.float64).reshape(n, 3),
             dimensions=np.array(dims, np.float64).reshape(n, 3),
             rotation_y=np.array(ry, np.float64).reshape(n),
             alpha=np.zeros(n) if alpha is None else np.array(alpha, np.float64))
    if score is not None:
        a['score'] = np.array(score, np.float64)
    else:
        a['occluded'] = np.zeros(n) if occluded is None else np.array(occluded, np.float64)
        a['truncated'] = np.zeros(n) if truncated is None else np.array(truncated, np.float64)
    return a


# ---------------------------------------------------------------------------- CPU
def test_oracle_reproduces_golden_counts():
    z, meta, gts, dts = load_golden()
    r = orc.evaluate(gts, dts, [0, 1, 2], [0, 1, 2], True, ke.MIN_OVERLAPS,
                     overlaps=golden_overlaps(z, gts, dts))
    assert np.array_equal(r['thr_count'], z['thr_count'])
    assert np.array_equal(r['thresholds'], z['thresholds'])
    assert np.array_equal(r['pr'][..., :3], z['pr'][..., :3])
    np.testing.assert_allclose(r['pr'][..., 3], z['pr'][..., 3], rtol=0, atol=1e-9)
    for c, s in enumerate(r['tp_scores']):
        assert np.array_equal(s, z['tp_scores'][z['tp_off'][c]:z['tp_off'][c + 1]])
    rets = {m: ke.precision_recall(r['pr'][m * 18:(m + 1) * 18], r['thr_count'][m * 18:],
                                   3, m == 0) for m in range(3)}
    for m in range(3):
        for n in ('precision', 'recall', 'orientation'):
            np.testing.assert_allclose(rets[m][n], z[n][m], rtol=0, atol=1e-12)
    result, ret_dict = ke.report([0, 1, 2], ['bbox', 'bev', '3d', 'aos'], True, rets)
    assert result == meta['result_str']
    assert {k: float('{:.4f}'.format(v)) for k, v in ret_dict.items()} == \
        {k: float('{:.4f}'.format(v)) for k, v in meta['ret_dict'].items()}


def test_oracle_overlaps_match_golden():
    z, _, gts, dts = load_golden()
    gov = golden_overlaps(z, gts, dts)
    for f in range(0, len(gts), 7):
        for m in range(3):
            o = orc.frame_overlaps(gts[f], dts[f], m)
            if m == 0:
                assert np.array_equal(o, gov[m][f])
            else:
                np.testing.assert_allclose(o, gov[m][f], rtol=0, atol=2e-6)


def test_invalid_inputs_raise_before_launch():
    g = anno(['Car'], [0, 0, 10, 50], [0, 1, 10], [4, 1.5, 1.6], [0])
    d = anno(['Car'], [0, 0, 10, 50], [0, 1, 10], [4, 1.5, 1.6], [0], score=[0.5])
    with pytest.raises(ValueError):
        ke.kitti_eval([g, g], [d], CLASSES)
    with pytest.raises(ValueError):
        ke.kitti_eval([g], [d], ['Van'])
    with pytest.raises(ValueError):
        ke.kitti_eval([g], [d], ['Truck'])
    with pytest.raises(ValueError):
        ke.kitti_eval([g], [d], CLASSES, eval_types=['aos'])
    with pytest.raises(ValueError):
        ke.kitti_eval([g], [{k: v for k, v in d.items() if k != 'score'}], CLASSES)
    with pytest.raises(ValueError):
        ke.kitti_eval([], [], CLASSES)


def test_class_ids():
    assert ke.class_ids('Car') == [0]
    assert ke.class_ids(['Cyclist', 1]) == [2, 1]


# ---------------------------------------------------------------------------- GPU
def device_rotate_iou(boxes, qboxes, criterion):
    import torch
    from depth_from_motion_b200 import capi
    b = torch.tensor(np.asarray(boxes, np.float32), device='cuda').contiguous()
    q = torch.tensor(np.asarray(qboxes, np.float32), device='cuda').contiguous()
    out = torch.empty(len(b), len(q), dtype=torch.float32, device='cuda')
    capi.check(capi.lib().dfm_op_eval_rotated_iou(
        ctypes.c_void_p(b.data_ptr()), ctypes.c_void_p(q.data_ptr()), len(b), len(q), criterion,
        ctypes.c_void_p(out.data_ptr()), None), 'dfm_op_eval_rotated_iou')
    torch.cuda.synchronize()
    return out.cpu().numpy()


def device_trig(boxes):
    """cosf / sinf of the yaws as the device computes them (torch's CUDA cos / sin call
    the same libdevice functions)"""
    return device_cos_sin(np.asarray(boxes, np.float32)[:, 4])


def device_cos_sin(yaw):
    import torch
    a = torch.tensor(np.asarray(yaw, np.float64).astype(np.float32), device='cuda')
    return torch.cos(a).cpu().numpy(), torch.sin(a).cpu().numpy()


def boundary_boxes():
    """axis-aligned and right-angle boxes placed on the 0.7 / 0.5 / 0.25 IoU boundaries, plus
    coincident boxes, boxes sharing an edge or a corner, and yaws of +-pi/2 and pi"""
    base = [0.0, 0.0, 4.0, 2.0]
    boxes, qboxes = [], []
    for t in (0.7, 0.5, 0.25):
        o = 8 * t / (1 + t)           # overlap length along x giving IoU t (l = 4, w = 2)
        for yaw in (0.0, math.pi, math.pi / 2, -math.pi / 2):
            sx = 4 - o
            if abs(yaw) == math.pi / 2:
                boxes.append([0, 0, 4, 2, yaw])
                qboxes.append([0, sx, 4, 2, yaw])
            else:
                boxes.append(base + [yaw])
                qboxes.append([sx, 0, 4, 2, yaw])
    for yaw in (0.0, math.pi / 2, -math.pi / 2, math.pi):
        boxes.append(base + [yaw])
        qboxes.append(base + [yaw])               # coincident
    boxes += [base + [0.0], base + [0.0], base + [0.0]]
    qboxes += [[4, 0, 4, 2, 0.0], [4, 2, 4, 2, 0.0], [0, 2, 4, 2, math.pi]]   # edge, corner
    return np.array(boxes, np.float32), np.array(qboxes, np.float32)


@pytest.mark.gpu
def test_rotated_iou_bitwise_at_boundaries():
    boxes, qboxes = boundary_boxes()
    # coincident boxes a half turn apart (yaw 0 against pi) intersect through corners a few
    # ulp apart, so the polygon depends on the last bit of sinf(pi): take the device's values
    tb, tq = device_trig(boxes), device_trig(qboxes)
    for crit in (-1, 0, 1, 2):
        dev = device_rotate_iou(boxes, qboxes, crit)
        ref = orc.rotate_iou_eval(boxes, qboxes, crit, trig=tb, qtrig=tq)
        assert np.array_equal(dev.view(np.uint32), ref.view(np.uint32)), (crit, dev - ref)
    diag = np.diag(device_rotate_iou(boxes, qboxes, -1))
    assert diag[12] == 1.0                     # coincident, yaw 0
    assert np.all(diag[16:18] == 0.0)          # shared edge / corner


@pytest.mark.gpu
def test_rotated_iou_bitwise_generic():
    rng = np.random.default_rng(3)
    n = 48
    boxes = np.stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(0.5, 5, n),
                      rng.uniform(0.5, 2.5, n), rng.uniform(-np.pi, np.pi, n)], 1)
    boxes = boxes.astype(np.float32)
    qboxes = boxes[rng.permutation(n)] + np.float32(0.3) * rng.standard_normal((n, 5)).astype(
        np.float32)
    tb, tq = device_trig(boxes), device_trig(qboxes)
    for crit in (-1, 2):
        dev = device_rotate_iou(boxes, qboxes, crit)
        ref = orc.rotate_iou_eval(boxes, qboxes, crit, trig=tb, qtrig=tq)
        assert np.array_equal(dev.view(np.uint32), ref.view(np.uint32))


def run_device(gts, dts, classes=(0, 1, 2), metrics=(0, 1, 2)):
    aos = ke.compute_aos_flag(gts, dts)
    ev = ke.KittiEvaluator(list(classes), list(metrics), aos)
    pr, cnt = ev.forward(ke.pack(gts, dts), keep=True)
    return ev, pr, cnt, aos


@pytest.mark.gpu
def test_golden_end_to_end():
    import torch
    z, meta, gts, dts = load_golden()
    ev, pr, cnt, aos = run_device(gts, dts)
    assert aos
    P = int(ke.pack(gts, dts)['pair_off'][-1])
    trig = [(device_cos_sin(d['rotation_y']), device_cos_sin(g['rotation_y']))
            for g, d in zip(gts, dts)]
    for m in range(3):
        o = ev.debug_tensor(f'overlap{m}', P, torch.float64)
        if m == 0:
            assert np.array_equal(o, z['overlap0'])
            continue
        # bitwise against the restatement given the device's cosf / sinf
        ref = np.concatenate([orc.frame_overlaps(g, d, m, t).reshape(-1)
                              for g, d, t in zip(gts, dts, trig)])
        assert np.array_equal(o, ref)
        # the golden comes from numba's simulator, whose cos / sin are float64: pairs with
        # nearly parallel edges amplify that last-bit difference of the corners (largest
        # observed: 1.3e-5 on 16 of 9891 pairs; the golden keeps every overlap 1e-4 away from
        # the min-overlaps it is compared with, so no matching decision depends on it)
        np.testing.assert_allclose(o, z[f'overlap{m}'], rtol=0, atol=2e-5)
        assert np.count_nonzero(np.abs(o - z[f'overlap{m}']) > 2e-6) <= 20
    assert np.array_equal(cnt, z['thr_count'])
    thr = ev.debug_tensor('thresholds', 54 * 41, torch.float64).reshape(54, 41)
    for c in range(54):
        assert np.array_equal(thr[c, :cnt[c]], z['thresholds'][c, :cnt[c]])
    S = 1 << max(0, int(len(np.concatenate([g['name'] for g in gts])) - 1).bit_length())
    tps = ev.debug_tensor('tp_scores', 54 * S, torch.float64).reshape(54, S)
    tpc = ev.debug_tensor('tp_count', 54, torch.int32)
    for c in range(54):
        assert np.array_equal(tps[c, :tpc[c]], z['tp_scores'][z['tp_off'][c]:z['tp_off'][c + 1]])
    assert np.array_equal(pr[..., :3], z['pr'][..., :3])
    np.testing.assert_allclose(pr[..., 3], z['pr'][..., 3], rtol=0, atol=1e-9)
    ev.close()
    result, ret_dict, inter = ke.kitti_eval(gts, dts, CLASSES, return_intermediates=True)
    for m in range(3):
        for n in ('precision', 'recall', 'orientation'):
            np.testing.assert_allclose(inter['rets'][m][n], z[n][m], rtol=0, atol=1e-12)
    assert result == meta['result_str']
    assert {k: float('{:.4f}'.format(v)) for k, v in ret_dict.items()} == \
        {k: float('{:.4f}'.format(v)) for k, v in meta['ret_dict'].items()}
    # determinism: a second run is bitwise equal
    result2, ret_dict2, inter2 = ke.kitti_eval(gts, dts, CLASSES, return_intermediates=True)
    assert np.array_equal(inter['pr'].view(np.uint64), inter2['pr'].view(np.uint64))
    assert result2 == result and ret_dict2 == ret_dict


def degenerate_frames():
    car = [4.0, 1.5, 1.6]
    gts, dts = [], []
    # 0: two cars, a van, a person_sitting, a DontCare; detections with a score tie, a box
    #    coincident with its GT, one under MIN_HEIGHT, one on a DontCare, yaws of +-pi/2, pi
    gts.append(anno(['Car', 'Car', 'Van', 'Person_sitting', 'DontCare', 'Pedestrian'],
                    [[100, 100, 200, 180], [300, 100, 400, 190], [500, 100, 620, 200],
                     [700, 100, 740, 200], [800, 100, 900, 200], [50, 200, 80, 260]],
                    [[0, 1, 10], [5, 1, 20], [-5, 1, 15], [8, 1, 12], [0, 1, 40], [2, 1, 8]],
                    [car, car, [5, 2, 2], [0.8, 1.2, 0.6], car, [0.8, 1.7, 0.6]],
                    [0, math.pi / 2, -math.pi / 2, math.pi, 0, 0],
                    alpha=[0.1, 0.2, 0.3, 0.4, -10, 0.5], occluded=[0, 1, 0, 0, -1, 2],
                    truncated=[0, 0.2, 0, 0, -1, 0.4]))
    dts.append(anno(['Car', 'Car', 'Car', 'Car', 'Car', 'Pedestrian', 'Pedestrian'],
                    [[100, 100, 200, 180], [102, 101, 201, 181], [300, 100, 400, 190],
                     [500, 100, 620, 200], [805, 100, 900, 120], [700, 100, 740, 200],
                     [50, 200, 80, 260]],
                    [[0, 1, 10], [0.1, 1, 10], [5, 1, 20.2], [-5, 1, 15], [0, 1, 40], [8, 1, 12],
                     [2, 1, 8]],
                    [car, car, car, [5, 2, 2], car, [0.8, 1.2, 0.6], [0.8, 1.7, 0.6]],
                    [0, 0, math.pi / 2, -math.pi / 2, 0, math.pi, 0],
                    alpha=[0.1, 0.0, 0.3, 0.2, 0, 0.4, 0.5],
                    score=[0.9, 0.9, 0.5, 0.7, 0.6, 0.8, 0.5]))
    # 1: no GT, two detections
    gts.append(anno([], np.zeros((0, 4)), np.zeros((0, 3)), np.zeros((0, 3)), []))
    dts.append(anno(['Car', 'Cyclist'], [[0, 0, 50, 60], [10, 10, 40, 80]],
                    [[1, 1, 10], [2, 1, 12]], [car, [1.7, 1.7, 0.6]], [0, 0],
                    score=[0.3, 0.4]))
    # 2: GT, no detections
    gts.append(anno(['Cyclist', 'Car'], [[0, 0, 50, 60], [100, 0, 150, 20]],
                    [[1, 1, 10], [5, 1, 30]], [[1.7, 1.7, 0.6], car], [0, 0]))
    dts.append(anno([], np.zeros((0, 4)), np.zeros((0, 3)), np.zeros((0, 3)), [], score=[]))
    # 3: only DontCare; a detection on it and one sharing its edge; a zero-height 2-D box
    gts.append(anno(['DontCare'], [[0, 0, 100, 100]], [[0, 1, 30]], [car], [0]))
    dts.append(anno(['Car', 'Car', 'Car'], [[0, 0, 100, 100], [100, 0, 200, 100],
                                             [10, 50, 90, 50]],
                    [[0, 1, 30], [4, 1, 30], [9, 1, 9]], [car, car, car], [0, 0, 0],
                    score=[0.5, 0.5, 0.5]))
    return gts, dts


def compare_with_oracle(gts, dts, classes=(0, 1, 2)):
    ev, pr, cnt, aos = run_device(gts, dts, classes)
    ev.close()
    r = orc.evaluate(gts, dts, list(classes), [0, 1, 2], aos, ke.MIN_OVERLAPS)
    assert np.array_equal(cnt, r['thr_count'])
    assert np.array_equal(pr[..., :3], r['pr'][..., :3])
    np.testing.assert_allclose(pr[..., 3], r['pr'][..., 3], rtol=0, atol=1e-12)
    return pr, cnt


@pytest.mark.gpu
def test_degenerate_frames_match_oracle():
    gts, dts = degenerate_frames()
    compare_with_oracle(gts, dts)
    result, ret_dict = ke.kitti_eval(gts, dts, CLASSES)
    assert all(np.isfinite(v) or np.isnan(v) for v in ret_dict.values())


@pytest.mark.gpu
def test_no_detections_anywhere():
    gts, dts = degenerate_frames()
    dts = [{k: v[:0] for k, v in d.items()} for d in dts]
    pr, cnt = compare_with_oracle(gts, dts)
    assert not cnt.any()
    _, ret_dict = ke.kitti_eval(gts, dts, CLASSES)
    assert all(v == 0 for v in ret_dict.values())
