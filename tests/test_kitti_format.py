"""KittiDataset's bbox2result_kitti / evaluate (depth_from_motion_b200.kitti_eval) against the
golden of the reference's own methods and box structures
(tests/golden/make_kitti_format_golden.py), the dfm_kitti_eval handle's conventions, and
DfM.simple_test -> evaluate end to end on the H100."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import kitti_eval as ke
from oracle import kitti_eval_oracle as orc

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
        'rotation_y', 'score', 'sample_idx')


def load():
    z = dict(np.load(os.path.join(GOLDEN, 'kitti_format.npz')))
    with open(os.path.join(GOLDEN, 'kitti_format.json')) as f:
        meta = json.load(f)
    nframes = len([k for k in z if k.endswith('_boxes_3d')])
    info = {'calib': {k: z[f'info_calib_{k}'] for k in ('P2', 'R0_rect', 'Tr_velo_to_cam')},
            'image': {'image_shape': z['info_image_shape']},
            'annos': {k[len('info_annos_'):]: v for k, v in z.items()
                      if k.startswith('info_annos_')}}
    infos = []
    for f in range(nframes):
        i = copy.deepcopy(info)
        i['image']['image_idx'] = 8 + f
        infos.append(i)
    results = [dict(boxes_3d=torch.from_numpy(z[f'in{f}_boxes_3d']),
                    scores_3d=torch.from_numpy(z[f'in{f}_scores_3d']),
                    labels_3d=torch.from_numpy(z[f'in{f}_labels_3d'])) for f in range(nframes)]
    return z, meta, infos, results


# ---------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('pseudo', [False, True])
def test_bbox2result_kitti_matches_golden(pseudo, tmp_path):
    z, meta, infos, results = load()
    annos = ke.bbox2result_kitti(results, infos, meta['classes'], meta['pcd_limit_range'],
                                 pseudo_lidar=pseudo, submission_prefix=str(tmp_path))
    for f, a in enumerate(annos):
        for k in KEYS:
            ref = z[f'out{int(pseudo)}_{f}_{k}']
            got = np.asarray(a[k])
            assert got.dtype == ref.dtype and got.shape == ref.shape, (f, k)
            assert np.array_equal(got, ref), (f, k)
    for i in infos:
        idx = i['image']['image_idx']
        assert (tmp_path / f'{idx:06d}.txt').read_text() == \
            meta['submission'][f'{int(pseudo)}_{idx:06d}']


def test_bbox2result_kitti_accepts_pts_bbox_and_refuses_2d_results():
    _, meta, infos, results = load()
    a = ke.bbox2result_kitti(results, infos, meta['classes'], pseudo_lidar=True)
    b = ke.bbox2result_kitti([{'pts_bbox': r} for r in results], infos, meta['classes'],
                             pseudo_lidar=True)
    for x, y in zip(a, b):
        assert all(np.array_equal(x[k], y[k]) for k in KEYS)
    with pytest.raises(ValueError):
        ke.bbox2result_kitti([np.zeros((1, 5))] * len(infos), infos, meta['classes'])
    with pytest.raises(ValueError):
        ke.bbox2result_kitti([{'img_bbox': r} for r in results], infos, meta['classes'])
    with pytest.raises(ValueError):
        ke.bbox2result_kitti(results[:-1], infos, meta['classes'])
    with pytest.raises(ValueError):
        ke.evaluate(results[:-1], infos, meta['classes'])


def test_more_than_three_classes_raise():
    with pytest.raises(ValueError):
        ke.class_ids(['Car', 'Pedestrian', 'Cyclist', 'Car'])


# ---------------------------------------------------------------------------- GPU
def _status_call(L, h, p, n_dt):
    """forward on one frame with one GT and n_dt detections (all zeros)"""
    dev = torch.device('cuda')
    gt = torch.zeros(1, 14, dtype=torch.float64, device=dev)
    dt = torch.zeros(n_dt, 13, dtype=torch.float64, device=dev)
    code = torch.zeros(max(n_dt, 1), dtype=torch.int32, device=dev)
    goff = torch.tensor([0, 1], dtype=torch.int32, device=dev)
    doff = torch.tensor([0, n_dt], dtype=torch.int32, device=dev)
    poff = torch.tensor([0, n_dt], dtype=torch.int64, device=dev)
    pr = torch.empty(18 * 41 * 4, dtype=torch.float64, device=dev)
    cnt = torch.empty(18, dtype=torch.int32, device=dev)
    st = torch.empty(1, dtype=torch.int32, device=dev)
    v = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = L.dfm_kitti_eval_forward(h, 1, 1, n_dt, n_dt, v(gt), v(code), v(goff), v(dt), v(code),
                                  v(doff), v(poff), v(pr), v(cnt), v(st), None)
    torch.cuda.synchronize()
    return rc, int(st.item())


@pytest.mark.gpu
def test_handle_contract():
    from depth_from_motion_b200 import capi
    L = capi.lib()
    ERR_INVALID, ERR_STATE = 1, 3
    d = capi.KittiEvalDesc()
    d.num_classes, d.num_metrics = 3, 1
    d.classes[0], d.classes[1], d.classes[2] = 0, 1, 2
    for i in range(18):
        d.min_overlap[i] = 0.5
    h = ctypes.c_void_p()
    capi.check(L.dfm_kitti_eval_create(ctypes.byref(d), ctypes.byref(h)), 'create')
    buf = torch.zeros(1 << 12, dtype=torch.float64, device='cuda')
    p = ctypes.c_void_p(buf.data_ptr())
    try:
        assert L.dfm_kitti_eval_debug_tensor(h, b'nope', p, 1, None) == ERR_INVALID
        assert L.dfm_kitti_eval_debug_tensor(h, b'thresholds', p, 18 * 41, None) == ERR_STATE
        assert L.dfm_kitti_eval_debug_tensor(h, b'overlap1', p, 1, None) == ERR_INVALID
        rc, status = _status_call(L, h, p, 4)
        assert rc == 0 and status == 0
        assert L.dfm_kitti_eval_debug_tensor(h, b'thresholds', p, 18 * 41, None) == 0
        assert L.dfm_kitti_eval_debug_tensor(h, b'thresholds', p, 18 * 41 + 1, None) == \
            ERR_INVALID
        assert L.dfm_kitti_eval_debug_tensor(h, b'overlap0', p, 4, None) == 0
        # a frame past the per-frame limit is refused through the status word
        rc, status = _status_call(L, h, p, ke.MAX_DT_PER_FRAME + 1)
        assert rc == 0 and status == 1
        rc, status = _status_call(L, h, p, ke.MAX_DT_PER_FRAME)
        assert rc == 0 and status == 0
    finally:
        L.dfm_kitti_eval_destroy(h)
    assert L.dfm_kitti_eval_destroy(None) == 0


@pytest.mark.gpu
def test_tie_break_decides_a_later_match():
    """Two detections of equal score both overlap GT 0; only the first (by index) also
    overlaps GT 1.  Index order gives GT 0 the first detection and leaves GT 1 unmatched (one
    TP); the other choice would give two TPs."""
    from tests.test_kitti_eval import anno
    car = [4.0, 1.5, 1.6]
    g = anno(['Car', 'Car'], [[0, 0, 100, 100], [10, 0, 110, 100]],
             [[0, 1, 10], [20, 1, 40]], [car, car], [0, 0])
    d = anno(['Car', 'Car'], [[5, 0, 105, 100], [-10, 0, 90, 100]],
             [[-20, 1, 60], [20, 1, 70]], [car, car], [0, 0], score=[0.8, 0.8])
    ev = ke.KittiEvaluator([0], [0], False)
    try:
        pr, cnt = ev.forward(ke.pack([g], [d]), keep=True)
        tpc = ev.debug_tensor('tp_count', 6, torch.int32)
    finally:
        ev.close()
    assert tpc[0] == 1     # bbox, Car, easy, overlap 0.7
    r = orc.evaluate([g], [d], [0], [0], False, ke.MIN_OVERLAPS)
    assert [len(s) for s in r['tp_scores']] == list(tpc)
    assert np.array_equal(pr[..., :3], r['pr'][..., :3]) and np.array_equal(cnt, r['thr_count'])


@pytest.mark.gpu
def test_too_many_detections_in_a_frame_raise():
    from tests.test_kitti_eval import anno
    n = ke.MAX_DT_PER_FRAME + 1
    g = anno(['Car'], [[0, 0, 100, 100]], [[0, 1, 10]], [[4, 1.5, 1.6]], [0])
    d = anno(['Car'] * n, np.tile([0, 0, 100, 100], (n, 1)), np.tile([0, 1, 10], (n, 1)),
             np.tile([4, 1.5, 1.6], (n, 1)), np.zeros(n), score=np.linspace(0, 1, n))
    with pytest.raises(ValueError):
        ke.kitti_eval([g], [d], 'Car')
    packed = ke.pack([g], [{k: v[:1] for k, v in d.items()}])
    packed.update(dt=np.tile(packed['dt'], (n, 1)), dt_code=np.tile(packed['dt_code'], n),
                  dt_off=np.array([0, n], np.int32), pair_off=np.array([0, n], np.int64))
    ev = ke.KittiEvaluator([0], [0], False)   # past the host check: the device refuses it
    try:
        with pytest.raises(RuntimeError):
            ev.forward(packed)
    finally:
        ev.close()


def device_cos_sin(yaw):
    a = torch.tensor(np.asarray(yaw, np.float64).astype(np.float32), device='cuda')
    return torch.cos(a).cpu().numpy(), torch.sin(a).cpu().numpy()


def oracle_ret_dict(gt_annos, dt_annos, classes):
    """kitti_eval's ret_dict through the host restatement (overlaps with the device's
    cosf / sinf, as the bitwise target)"""
    ids = ke.class_ids(classes)
    aos = ke.compute_aos_flag(gt_annos, dt_annos)
    ovs = {m: [orc.frame_overlaps(g, d, m, (device_cos_sin(d['rotation_y']),
                                            device_cos_sin(g['rotation_y'])))
               for g, d in zip(gt_annos, dt_annos)] for m in range(3)}
    r = orc.evaluate(gt_annos, dt_annos, ids, [0, 1, 2], aos, ke.MIN_OVERLAPS, overlaps=ovs)
    per = len(ids) * 6
    rets = {m: ke.precision_recall(r['pr'][m * per:(m + 1) * per],
                                   r['thr_count'][m * per:(m + 1) * per], len(ids), m == 0 and aos)
            for m in range(3)}
    eval_types = ['bbox', 'bev', '3d'] + (['aos'] if aos else [])
    return ke.report(ids, eval_types, aos, rets), r


def _check_evaluate(results, infos, classes, pseudo):
    dt_annos = ke.bbox2result_kitti(results, infos, classes, pseudo_lidar=pseudo)
    gt_annos = [i['annos'] for i in infos]
    (ref_str, ref_dict), r = oracle_ret_dict(gt_annos, dt_annos, classes)
    _, got_dict, inter = ke.kitti_eval(gt_annos, dt_annos, classes, return_intermediates=True)
    assert np.array_equal(inter['thr_count'], r['thr_count'])
    assert np.array_equal(inter['pr'][..., :3], r['pr'][..., :3])
    plain, got_str = ke.evaluate(results, infos, classes, pseudo_lidar=pseudo, return_str=True)
    assert got_str == ref_str
    assert plain.keys() == ref_dict.keys()
    assert all(plain[k] == ref_dict[k] or (np.isnan(plain[k]) and np.isnan(ref_dict[k]))
               for k in plain)
    wrapped = ke.evaluate([{'pts_bbox': x} for x in results], infos, classes,
                          pseudo_lidar=pseudo)
    assert wrapped == {f'pts_bbox/{k}': float('{:.4f}'.format(v)) for k, v in ref_dict.items()}
    return dt_annos


@pytest.mark.gpu
def test_evaluate_matches_oracle_on_golden_boxes():
    _, meta, infos, results = load()
    for pseudo in (False, True):
        _check_evaluate(results, infos, meta['classes'], pseudo)


@pytest.mark.gpu
def test_dfm_simple_test_to_evaluate():
    from tests.test_detector import KITTI, _cuda_detector, _free, _kitti_inputs
    _, _, infos, _ = load()
    det = _cuda_detector(KITTI, 0)
    try:
        results = []
        for seed in range(len(infos)):
            img, metas = _kitti_inputs(seed)
            results += det.simple_test(img, metas)
    finally:
        _free(det)
    assert all(r['boxes_3d'].device.type == 'cpu' for r in results)
    _check_evaluate(results, infos, ['Car', 'Pedestrian', 'Cyclist'], True)
