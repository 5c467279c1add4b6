"""WaymoDataset's KITTI metric for load_mode 'lidar_frame' (depth_from_motion_b200.waymo_eval:
convert_valid_bboxes / bbox2result_kitti / evaluate, dfm_waymo_kitti_convert) against the
golden of the reference's own methods and kitti_eval (tests/golden/make_waymo_kitti_golden.py),
and the KITTI evaluator's frame parts at Waymo-val size."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import kitti_eval as ke
from depth_from_motion_b200 import waymo_eval as we
from oracle import waymo_kitti_oracle as orc

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
        'rotation_y', 'score', 'sample_idx')
GT_KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
           'rotation_y')


def load():
    z = dict(np.load(os.path.join(GOLDEN, 'waymo_kitti.npz')))
    with open(os.path.join(GOLDEN, 'waymo_kitti.json')) as f:
        meta = json.load(f)
    infos, results = [], []
    for f in range(meta['num_frames']):
        infos.append({'calib': {k: z[f'info_calib_{k}'] for k in ('P0', 'R0_rect',
                                                                   'Tr_velo_to_cam')},
                      'image': {'image_shape': z['info_image_shape'],
                                'image_idx': int(z['info_image_idx'][f])},
                      # replaced by cam_sync_annos when cam_sync is set
                      'annos': {k: z[f'gt0_{k}'][:1] for k in GT_KEYS},
                      'cam_sync_annos': {k: z[f'gt{f}_{k}'] for k in GT_KEYS}})
        results.append(dict(boxes_3d=torch.from_numpy(z[f'in{f}_boxes_3d']),
                            scores_3d=torch.from_numpy(z[f'in{f}_scores_3d']),
                            labels_3d=torch.from_numpy(z[f'in{f}_labels_3d'])))
    return z, meta, infos, results


# ---------------------------------------------------------------------------- CPU
def test_oracle_reproduces_golden_annos_and_submission(tmp_path):
    z, meta, infos, results = load()
    annos = orc.bbox2result_kitti(results, infos, meta['classes'],
                                  submission_prefix=str(tmp_path))
    for f, a in enumerate(annos):
        for k in KEYS:
            ref, got = z[f'out{f}_{k}'], np.asarray(a[k])
            assert got.dtype == ref.dtype and got.shape == ref.shape, (f, k)
            assert np.array_equal(got, ref), (f, k)
    written = {p.name: p.read_text() for p in tmp_path.iterdir()}
    assert written == meta['submission']
    # frames that keep nothing write no file
    assert len(written) == sum(len(a['name']) > 0 for a in annos) < len(annos)


def test_golden_covers_the_cases():
    z, meta, infos, _ = load()
    n_gt = [len(z[f'gt{f}_name']) for f in range(meta['num_frames'])]
    assert max(n_gt) >= 100 and min(n_gt) == 0
    assert any('Sign' in z[f'gt{f}_name'] for f in range(meta['num_frames']))
    boxes = np.concatenate([z[f'in{f}_boxes_3d'] for f in range(meta['num_frames'])])
    lim = np.array(meta['pcd_limit_range'])
    inside = ((boxes[:, :3] > lim[:3]) & (boxes[:, :3] < lim[3:])).all(1)
    assert inside.any() and (~inside).any()
    assert (boxes[inside, 0] < 0).any()                   # behind the FRONT camera
    assert (np.abs(boxes[:, 6]) > np.pi).any()            # yaws past +-pi


def test_cam_sync_annos_are_chosen():
    _, _, infos, _ = load()
    assert we.gt_annos_of(infos)[0] is infos[0]['cam_sync_annos']
    assert we.gt_annos_of(infos, cam_sync=False)[0] is infos[0]['annos']
    bad = copy.deepcopy(infos)
    del bad[3]['cam_sync_annos']
    with pytest.raises(ValueError):
        we.gt_annos_of(bad)


def test_evaluate_key_and_rounding_rules(monkeypatch):
    _, _, infos, results = load()
    seen = []

    def fake_score(res, data_infos, class_names, limit, gt, eval_types, prefix, limit_bytes):
        seen.append((eval_types, prefix, gt['off'][-1]))
        return 'report', {'KITTI/Car_3D_AP11_easy_strict': 12.345678,
                          'Car_BEV_AP40_hard_loose': 1 / 3}

    monkeypatch.setattr(we, '_score', fake_score)
    plain = we.evaluate(results, infos)
    assert plain == {'KITTI/Car_3D_AP11_easy_strict': 12.345678, 'Car_BEV_AP40_hard_loose': 1 / 3}
    assert seen[-1][0] == ['bbox', 'bev', '3d'] and seen[-1][1] is None
    n_cam_sync = sum(len(i['cam_sync_annos']['name']) for i in infos)
    assert seen[-1][2] == n_cam_sync
    wrapped, s = we.evaluate([{'pts_bbox': r} for r in results], infos, submission_prefix='x/',
                             return_str=True)
    assert wrapped == {'pts_bbox/KITTI/Car_3D_AP11_easy_strict': 12.3457,
                       'pts_bbox/Car_BEV_AP40_hard_loose': 0.3333}
    assert seen[-1][0] == ['bev', '3d'] and seen[-1][1] == 'x/pts_bbox'
    assert s.startswith('Results of pts_bbox:')
    we.evaluate(results, infos, cam_sync=False)
    assert seen[-1][2] == len(infos)


def test_default_class_names_follow_the_multiview_dfm_configs(monkeypatch):
    """Both MultiViewDfM configs set class_names = ['Pedestrian', 'Cyclist', 'Car']; that is
    WaymoDataset.CLASSES, so simple_test's label 0 is a pedestrian."""
    _, _, infos, results = load()
    assert we.WAYMO_CLASSES == ('Pedestrian', 'Cyclist', 'Car')
    seen = []
    monkeypatch.setattr(we, '_score', lambda res, di, class_names, *a: (
        seen.append(list(class_names)) or ('', {})))
    we.evaluate(results, infos)
    assert seen == [['Pedestrian', 'Cyclist', 'Car']]
    c = dict(off=np.array([0, 3]), keep=np.ones(3, bool), out=np.zeros((3, we.CONVERT_W),
                                                                      np.float32),
             labels=np.array([0, 1, 2]), scores=np.ones(3, np.float32),
             sample_idx=np.zeros(3, np.int64))
    cols, off = we._kept_columns(c, we.WAYMO_CLASSES)
    assert list(cols['name']) == ['Pedestrian', 'Cyclist', 'Car']
    assert list(cols['code']) == [1, 2, 0]     # the evaluator's Pedestrian, Cyclist, Car
    assert list(off) == [0, 3]


def test_kept_offsets_with_empty_and_dropped_frames():
    c = dict(off=np.array([0, 2, 2, 5, 5]), keep=np.array([1, 0, 0, 1, 1], bool),
             out=np.zeros((5, we.CONVERT_W), np.float32), labels=np.zeros(5, np.int64),
             scores=np.ones(5, np.float32), sample_idx=np.zeros(5, np.int64))
    _, off = we._kept_columns(c, we.WAYMO_CLASSES)
    assert list(off) == [0, 1, 1, 3, 3]


def test_bad_inputs_raise():
    _, meta, infos, results = load()
    with pytest.raises(NotImplementedError, match='write_objects'):
        we.evaluate(results, infos, metric='waymo')
    with pytest.raises(NotImplementedError):
        we.evaluate(results, infos, metric=['kitti', 'waymo'])
    with pytest.raises(ValueError):
        we.evaluate(results, infos, metric='nuscenes')
    with pytest.raises(ValueError):
        we.evaluate(results[:-1], infos)
    with pytest.raises(ValueError):
        we.evaluate([{'img_bbox2d': r} for r in results], infos)
    with pytest.raises(ValueError):
        we.convert_set(results[:-1], infos)
    with pytest.raises(ValueError):
        orc.bbox2result_kitti(results[:-1], infos, meta['classes'])
    # the column path refuses what pack refuses
    gt = ke.concat_annos([i['cam_sync_annos'] for i in infos], ('name',) + ke.GT_COLS)
    dt = ke.concat_annos(orc.bbox2result_kitti(results, infos, meta['classes']),
                         ('name',) + ke.DT_COLS)
    with pytest.raises(ValueError):
        ke.pack_columns(gt, dict(dt, off=dt['off'][:-1]))
    with pytest.raises(ValueError):
        ke.pack_columns(gt, dict(dt, off=dt['off'][::-1]))
    with pytest.raises(ValueError):
        ke.pack_columns(gt, dict(dt, bbox=dt['bbox'][:-1]))


def test_column_packing_equals_per_frame_packing():
    _, meta, infos, results = load()
    gts = [i['cam_sync_annos'] for i in infos]
    dts = orc.bbox2result_kitti(results, infos, meta['classes'])
    a = ke.pack(gts, dts)
    gt = ke.concat_annos(gts, ('name',) + ke.GT_COLS)
    dt = ke.concat_annos(dts, ('name',) + ke.DT_COLS)
    b = ke.pack_columns(gt, dt)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert ke.compute_aos_flag(gts, dts) == ke.compute_aos_flag_columns(gt, dt)
    # names compare lower-cased; only the exact 'DontCare' is DontCare
    assert list(ke.name_codes(np.array(['car', 'CAR', 'Van', 'DontCare', 'dontcare', 'Sign']),
                              True)) == [0, 0, 3, 7 | 8, 7, 7]


# ---------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_device_conversion_matches_golden():
    z, meta, infos, results = load()
    annos = we.bbox2result_kitti(results, infos, meta['classes'])
    ref_annos = orc.bbox2result_kitti(results, infos, meta['classes'])
    for f, (a, r) in enumerate(zip(annos, ref_annos)):
        for k in KEYS:
            gold, got = z[f'out{f}_{k}'], np.asarray(a[k])
            assert got.dtype == gold.dtype and got.shape == gold.shape, (f, k)
            if k in ('name', 'truncated', 'occluded', 'score', 'sample_idx', 'dimensions'):
                assert np.array_equal(got, gold), (f, k)
            else:
                # BLAS sums and libm / libdevice trigonometry: float32 rounding of the oracle.
                # A corner near the camera plane divides by a small depth, which magnifies
                # that rounding in the 2-D box (up to 2e-5 relative, at |x| ~ 1e6 px)
                rtol = 1e-4 if k == 'bbox' else 2e-6
                np.testing.assert_allclose(got, r[k], rtol=rtol, atol=2e-5, err_msg=f'{f} {k}')
                np.testing.assert_allclose(got, gold, rtol=rtol, atol=2e-5, err_msg=f'{f} {k}')
                if k == 'bbox':
                    near = np.abs(gold) < 1e4
                    np.testing.assert_allclose(got[near], gold[near], rtol=2e-6, atol=2e-5)
    # the keep masks exactly; per-frame convert_valid_bboxes against the oracle
    for res, info in zip(results, infos):
        got = we.convert_valid_bboxes(res, info)
        ref = orc.convert_valid_bboxes(res, info)
        for k in ('bbox', 'box3d_camera', 'box3d_lidar', 'scores', 'label_preds'):
            assert got[k].shape == ref[k].shape and got[k].dtype == ref[k].dtype, k
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-4 if k == 'bbox' else 2e-6,
                                       atol=2e-5, err_msg=k)
        assert got['sample_idx'] == ref['sample_idx']


@pytest.mark.gpu
def test_device_conversion_refuses_labels_without_names():
    _, meta, infos, results = load()
    bad = [dict(r, labels_3d=r['labels_3d'] + 3) for r in results]
    with pytest.raises(ValueError):
        we.bbox2result_kitti(bad, infos, meta['classes'])


@pytest.mark.gpu
def test_evaluate_matches_golden(tmp_path):
    _, meta, infos, results = load()
    got, got_str = we.evaluate(results, infos, meta['classes'], return_str=True,
                               submission_prefix=str(tmp_path / 'sub'))
    ref = meta['plain']['ret_dict']
    assert got.keys() == ref.keys()
    assert {k: float('{:.4f}'.format(v)) for k, v in got.items()} == \
        {k: float('{:.4f}'.format(v)) for k, v in ref.items()}
    assert got_str == meta['plain']['result_str']
    assert sorted(p.name for p in (tmp_path / 'sub').iterdir()) == sorted(meta['submission'])
    # wrapped: BEV and 3-D on the frames with GT, whose alphas are -10
    frames = meta['pts_bbox']['frames']
    sub_infos = [copy.deepcopy(infos[f]) for f in frames]
    for i in sub_infos:
        i['cam_sync_annos']['alpha'] = np.full(len(i['cam_sync_annos']['alpha']), -10.0)
    wrapped = we.evaluate([{'pts_bbox': results[f]} for f in frames], sub_infos,
                          meta['classes'])
    assert wrapped == meta['pts_bbox']['ret_dict']
    # with valid alphas the reference fails on BEV / 3-D alone; so does this
    with pytest.raises(ValueError):
        we.evaluate([{'pts_bbox': results[f]} for f in frames], [infos[f] for f in frames])


def waymo_val_columns(frames=39987, dt_per_frame=500, seed=0):
    """A synthetic set of Waymo-val size in column form: 50-300 GT per frame (Car,
    Pedestrian, Cyclist, Sign), detections jittered from the frame's GT, GT alphas -10."""
    rng = np.random.default_rng(seed)
    ng = rng.integers(50, 301, frames)
    G = int(ng.sum())
    g_off = np.concatenate([[0], np.cumsum(ng)])
    names = np.array(['Car', 'Pedestrian', 'Cyclist', 'Sign'])
    loc = np.stack([rng.uniform(-40, 40, G), rng.uniform(1, 2, G), rng.uniform(2, 80, G)], 1)
    dims = np.stack([rng.uniform(0.5, 5, G), rng.uniform(1.4, 2, G), rng.uniform(0.5, 2, G)], 1)
    x0, y0 = rng.uniform(0, 1800, G), rng.uniform(300, 900, G)
    bbox = np.stack([x0, y0, x0 + rng.uniform(10, 300, G), y0 + rng.uniform(20, 200, G)], 1)
    ry = rng.uniform(-np.pi, np.pi, G)
    gt = dict(off=g_off, name=names[rng.choice(4, G, p=(0.5, 0.3, 0.1, 0.1))],
              alpha=np.full(G, -10.0), bbox=bbox, location=loc, dimensions=dims, rotation_y=ry,
              occluded=rng.integers(0, 3, G).astype(np.float64),
              truncated=rng.choice([0.0, 0.2, 0.4], G))
    D = frames * dt_per_frame
    d_frame = np.repeat(np.arange(frames), dt_per_frame)
    src = g_off[d_frame] + rng.integers(0, ng[d_frame])
    sig = rng.uniform(0.02, 1.0, D)[:, None].astype(np.float32)
    f32 = lambda a: a.astype(np.float32)
    dt = dict(off=np.arange(frames + 1) * dt_per_frame,
              name=names[rng.integers(0, 3, D)],
              alpha=f32(rng.uniform(-np.pi, np.pi, D)),
              bbox=f32(bbox[src] + rng.normal(0, 6, (D, 4)) * sig),
              location=f32(loc[src] + rng.normal(0, 0.6, (D, 3)) * sig),
              dimensions=f32(dims[src] * (1 + rng.normal(0, 0.05, (D, 3)))),
              rotation_y=f32(ry[src] + rng.normal(0, 0.2, D)),
              score=f32(rng.uniform(0, 1, D)))
    return gt, dt


@pytest.mark.gpu
def test_parts_are_bitwise_equal_at_waymo_val_size():
    gt, dt = waymo_val_columns()
    packed = ke.pack_columns(gt, dt)
    P = int(packed['pair_off'][-1])
    out = {}
    for name, limit in (('one', 2 * P * 8), ('parts', 1 << 30)):
        ev = ke.KittiEvaluator([0, 1, 2], [1, 2], False, overlap_limit=limit)
        try:
            pr, cnt = ev.forward(packed)
            ws, ov, parts = ev.workspace()
        finally:
            ev.close()
        assert ov <= limit
        out[name] = (pr, cnt, parts, ws)
        torch.cuda.empty_cache()
    assert out['one'][2] == 1 and out['parts'][2] > 20
    assert np.array_equal(out['one'][0].view(np.uint64), out['parts'][0].view(np.uint64))
    assert np.array_equal(out['one'][1], out['parts'][1])
    assert out['parts'][1].max() > 1                      # thresholds were found
    # the part-independent workspace is O(frames + GT + detections)
    assert out['parts'][3] - (1 << 30) < 64 * (len(packed['gt']) + len(packed['dt']) +
                                                 41 * (len(gt['off']) - 1)) * 8


def _forward(packed, metrics, aos, limit):
    ev = ke.KittiEvaluator([0, 1, 2], metrics, aos, overlap_limit=limit)
    try:
        pr, cnt = ev.forward(packed, keep=True)
        nc = len(metrics) * 18
        thr = ev.debug_tensor('thresholds', nc * 41, torch.float64)
        return pr, cnt, thr, ev.workspace()
    finally:
        ev.close()


@pytest.mark.gpu
def test_parts_are_bitwise_equal_with_bbox_and_aos():
    """bbox, BEV and 3-D with AOS (what plain Waymo results take) in one part and in parts of
    a few frames: counts, thresholds and similarity sums bitwise equal."""
    gt, dt = waymo_val_columns(frames=400, dt_per_frame=100, seed=1)
    gt['alpha'] = np.random.default_rng(2).uniform(-np.pi, np.pi, len(gt['alpha']))
    assert ke.compute_aos_flag_columns(gt, dt)
    packed = ke.pack_columns(gt, dt)
    P = int(packed['pair_off'][-1])
    one = _forward(packed, [0, 1, 2], True, 3 * P * 8)
    parts = _forward(packed, [0, 1, 2], True, 3 * 8 * 4 * 300 * 100)
    assert one[3][2] == 1 and parts[3][2] > 50
    assert (one[0][:18, :, 3] != 0).any()                   # AOS similarities were summed
    for a, b in zip(one[:3], parts[:3]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    # and through evaluate on the golden set, in parts of a few frames
    _, meta, infos, results = load()
    ref = we.evaluate(results, infos, meta['classes'])
    assert we.evaluate(results, infos, meta['classes'], overlap_limit=3 * 8 * 130 * 130) == ref


@pytest.mark.gpu
def test_overlap_limit_is_checked():
    from depth_from_motion_b200 import capi
    ev = ke.KittiEvaluator([0], [1], False, overlap_limit=4)
    with pytest.raises(RuntimeError):
        ev._handle(0)
    ev.close()
    gt, dt = waymo_val_columns(frames=3, dt_per_frame=20)
    packed = ke.pack_columns(gt, dt)
    small = int(np.diff(packed['pair_off']).max()) * 8 - 8   # below one frame's overlaps
    ev = ke.KittiEvaluator([0], [1], False, overlap_limit=small)
    try:
        with pytest.raises(RuntimeError, match='overlap limit'):
            ev.forward(packed)
    finally:
        ev.close()
    assert capi.lib().dfm_kitti_eval_set_overlap_limit(None, 1 << 20) != 0
