"""Writes tests/golden/waymo_kitti.npz + waymo_kitti.json: WaymoDataset's KITTI metric for
load_mode 'lidar_frame' (mmdet3d datasets/waymo_dataset.py).  WaymoDataset.convert_valid_bboxes
and bbox2result_kitti run verbatim through oracle/ref_loader with the reference's own box
structures (mmcv stubbed, as in make_kitti_format_golden.py), and kitti_eval runs verbatim
under numba's CUDA simulator (as in make_kitti_eval_golden.py).

Input: 12 frames on the calibration and image shape of the reference's
tests/data/waymo/kitti_format/waymo_infos_val.pkl (image_idx changed per frame), with
synthetic cam_sync_annos: GT LiDAR boxes of Car / Pedestrian / Cyclist / Sign converted to
camera annos by the reference's convert_valid_bboxes; two frames hold 100+ GT boxes, one holds
none.  Detections are jittered GT boxes and false positives, inside and outside the
[-85, -85, -5, 85, 85, 5] range, behind the FRONT camera, with yaws past +-pi, and one
frame has none.  Detections whose centre lies within 1e-4 of a range edge, or whose overlap
with a GT lies within 1e-4 of a min-overlap, are dropped, so no decision depends on the last
bits of the projection or of the simulator's float64 trigonometry.

Stored: the inputs, every array of the KITTI-format annos and the submission text, and
kitti_eval's ret_dict and result string for plain results (default eval types) and for
results wrapped as {'pts_bbox': ...} (eval_types ['bev', '3d'], on the GT with every alpha set
to -10: with valid alphas the reference's kitti_eval fails for these eval types, and it is recorded on the
frames that hold GT).

Run from the repository root: python tests/golden/make_waymo_kitti_golden.py
"""
import ast
import copy
import importlib.util
import json
import os
import pickle
import sys
import tempfile

os.environ['NUMBA_ENABLE_CUDASIM'] = '1'
import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from oracle import ref_loader as rl  # noqa: E402

CLASSES = ['Car', 'Pedestrian', 'Cyclist']
GT_NAMES = ('Car', 'Pedestrian', 'Cyclist', 'Sign')
PCD_LIMIT_RANGE = [-85, -85, -5, 85, 85, 5]
KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
        'rotation_y', 'score', 'sample_idx')
GT_KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
           'rotation_y')
MIN_OVERLAPS = (0.7, 0.5, 0.25)
MARGIN = 1e-4
NUM_FRAMES = 12


def _sibling(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def waymo_methods(namespace):
    """WaymoDataset.convert_valid_bboxes / bbox2result_kitti, their source unchanged."""
    path = os.path.join(rl.REFERENCE_ROOT, 'mmdet3d/datasets/waymo_dataset.py')
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body
               if isinstance(n, ast.ClassDef) and n.name == 'WaymoDataset')
    out = {}
    for fn in cls.body:
        if isinstance(fn, ast.FunctionDef) and fn.name in ('convert_valid_bboxes',
                                                          'bbox2result_kitti'):
            code = ast.get_source_segment(src, fn)
            code = '\n'.join(l[4:] if l.startswith('    ') else l for l in code.split('\n'))
            exec(compile(code, path, 'exec'), namespace)
            out[fn.name] = namespace[fn.name]
    return out


def lidar_boxes(rng, n, names):
    """n LiDAR boxes (bottom centre) sized by class, spread around the FRONT camera."""
    size = {'Car': (4.5, 2.0, 1.7), 'Pedestrian': (0.9, 0.9, 1.8), 'Cyclist': (1.8, 0.8, 1.7),
            'Sign': (0.3, 0.8, 0.8)}
    base = np.array([size[str(x)] for x in names]).reshape(n, 3)
    x = rng.uniform(-20, 80, n)       # x < 0: behind the FRONT camera
    y = rng.uniform(-40, 40, n)
    z = rng.uniform(-2.5, 0.5, n)
    dims = base * rng.uniform(0.8, 1.2, (n, 3))
    yaw = rng.uniform(-4, 4, n)       # limit_yaw folds these into [-pi, pi)
    return np.concatenate([np.stack([x, y, z], 1), dims, yaw[:, None]], 1)


def main():
    fmt = _sibling('make_kitti_format_golden')
    LiDARBoxes, Box3DMode, points_cam2img = fmt.load_structures()
    ns = dict(np=np, torch=torch, mmcv=fmt._Mmcv, Box3DMode=Box3DMode,
              points_cam2img=points_cam2img)
    methods = waymo_methods(ns)
    ev = _sibling('make_kitti_eval_golden').load_eval()
    with open(os.path.join(rl.REFERENCE_ROOT,
                           'tests/data/waymo/kitti_format/waymo_infos_val.pkl'), 'rb') as f:
        base = pickle.load(f)[0]
    rng = np.random.default_rng(0)

    def dataset(infos):
        ds = type('Dataset', (), {})()
        ds.load_mode, ds.pcd_limit_range, ds.data_infos = 'lidar_frame', PCD_LIMIT_RANGE, infos
        ds.convert_valid_bboxes = methods['convert_valid_bboxes'].__get__(ds)
        return ds

    def convert(boxes, scores, labels, infos):
        wrapped = [dict(boxes_3d=LiDARBoxes(torch.tensor(b, dtype=torch.float32)),
                        scores_3d=torch.tensor(s, dtype=torch.float32),
                        labels_3d=torch.tensor(l, dtype=torch.int64))
                   for b, s, l in zip(boxes, scores, labels)]
        return methods['bbox2result_kitti'](dataset(infos), wrapped, list(GT_NAMES))

    infos, gt_boxes, gt_labels = [], [], []
    for f in range(NUM_FRAMES):
        i = {k: copy.deepcopy(base[k]) for k in ('image', 'calib')}
        i['image']['image_idx'] = 1000000 + 7 * f
        infos.append(i)
        n = 0 if f == 4 else (int(rng.integers(100, 130)) if f in (1, 8) else
                              int(rng.integers(5, 30)))
        lab = rng.choice(4, n, p=(0.55, 0.25, 0.1, 0.1))
        b = lidar_boxes(rng, n, np.array(GT_NAMES)[lab])
        b[:, 0] = np.where(np.abs(b[:, 0]) > 70, rng.uniform(5, 60, n), b[:, 0])   # in range
        gt_boxes.append(b)
        gt_labels.append(lab)
    # GT: the reference's own conversion of the GT LiDAR boxes, with KITTI difficulty fields
    gts = convert(gt_boxes, [np.ones(len(b)) for b in gt_boxes], gt_labels, infos)
    for g in gts:
        n = len(g['name'])
        g['occluded'] = rng.integers(0, 3, n).astype(np.int64) if n else np.array([], np.int64)
        g['truncated'] = rng.choice((0.0, 0.2, 0.4), n) if n else np.array([])
        for k in ('alpha', 'bbox', 'dimensions', 'location', 'rotation_y', 'truncated'):
            g[k] = np.asarray(g[k], np.float64)   # as waymo_infos_*.pkl store them
        g.pop('score')
        g.pop('sample_idx')
    # detections: jittered GT boxes (some relabelled) and false positives
    boxes, scores, labels = [], [], []
    for f in range(NUM_FRAMES):
        g, gl = gt_boxes[f], gt_labels[f]
        src = np.flatnonzero((gl < 3) & (rng.uniform(size=len(gl)) > 0.2))
        nfp = int(rng.integers(2, 12))
        sig = rng.uniform(0.02, 0.5, len(src))[:, None]
        tp = g[src] + rng.normal(0, 1, (len(src), 7)) * sig * [1, 1, 0.3, 0.3, 0.3, 0.3, 1]
        lab = np.where(rng.uniform(size=len(src)) < 0.9, gl[src], rng.integers(0, 3, len(src)))
        fp_lab = rng.integers(0, 3, nfp)
        fp = lidar_boxes(rng, nfp, np.array(GT_NAMES)[fp_lab])
        fp[:, :2] += rng.choice((0, 1), (nfp, 1)) * rng.choice((-80, 80), (nfp, 2))   # out
        b = np.concatenate([tp, fp])
        l = np.concatenate([lab, fp_lab]).astype(np.int64)
        s = rng.uniform(0, 1, len(b)).round(3)
        if f == 6:
            b, l, s = b[:0], l[:0], s[:0]
        boxes.append(b.astype(np.float32))
        labels.append(l)
        scores.append(s.astype(np.float32))

    def near_edge(b):
        c = b[:, :3]
        lo, hi = np.array(PCD_LIMIT_RANGE[:3]), np.array(PCD_LIMIT_RANGE[3:])
        return np.any((np.abs(c - lo) < MARGIN) | (np.abs(c - hi) < MARGIN), axis=1)

    while True:
        dts = convert(boxes, scores, labels, infos)
        dts = [{k: v for k, v in d.items()} for d in dts]
        for d in dts:
            d['name'] = np.asarray([CLASSES[GT_NAMES.index(str(x))] for x in d['name']],
                                   '<U10') if len(d['name']) else d['name']
        # map each kept detection back to its input row
        bad = {}
        for f in range(NUM_FRAMES):
            b = boxes[f]
            lr = np.array(PCD_LIMIT_RANGE, np.float32)
            keep = np.flatnonzero(((b[:, :3] > lr[:3]) & (b[:, :3] < lr[3:])).all(1))
            drop = set(np.flatnonzero(near_edge(b)).tolist())
            for metric in range(3):
                if len(dts[f]['name']) and len(gts[f]['name']):
                    ov = ev.calculate_iou_partly([dts[f]], [gts[f]], metric, 1)[0][0]
                    for j in np.flatnonzero(np.any(np.abs(ov[..., None] - MIN_OVERLAPS) <
                                                   MARGIN, axis=(1, 2))):
                        drop.add(int(keep[j]))
            if drop:
                bad[f] = sorted(drop)
        if not bad:
            break
        for f, rows in bad.items():
            m = np.ones(len(boxes[f]), bool)
            m[rows] = False
            boxes[f], labels[f], scores[f] = boxes[f][m], labels[f][m], scores[f][m]

    arrays, texts = {}, {}
    for f in range(NUM_FRAMES):
        arrays[f'in{f}_boxes_3d'], arrays[f'in{f}_scores_3d'] = boxes[f], scores[f]
        arrays[f'in{f}_labels_3d'] = labels[f]
        for k in GT_KEYS:
            arrays[f'gt{f}_{k}'] = gts[f][k]
    wrapped = [dict(boxes_3d=LiDARBoxes(torch.tensor(b)), scores_3d=torch.tensor(s),
                    labels_3d=torch.tensor(l)) for b, s, l in zip(boxes, scores, labels)]
    with tempfile.TemporaryDirectory() as tmp:
        annos = methods['bbox2result_kitti'](dataset(infos), wrapped, CLASSES, None, tmp)
        for name in sorted(os.listdir(tmp)):
            with open(os.path.join(tmp, name)) as fh:
                texts[name] = fh.read()
    for f, a in enumerate(annos):
        for k in KEYS:
            arrays[f'out{f}_{k}'] = np.asarray(a[k])
    plain_str, plain = ev.kitti_eval(gts, annos, CLASSES)
    # with eval_types ['bev', '3d'] the reference fails (a None mAP_aos) wherever AOS is
    # valid, so the wrapped case is recorded on GT whose alphas are -10
    # (and a GT frame without boxes makes it read past an empty alpha): the frames with GT
    wrapped_frames = [f for f in range(NUM_FRAMES) if len(gts[f]['name'])]
    gts_noalpha = [dict(gts[f], alpha=np.full(len(gts[f]['alpha']), -10.0))
                   for f in wrapped_frames]
    wrapped_str, wrapped_d = ev.kitti_eval(gts_noalpha, [annos[f] for f in wrapped_frames],
                                           CLASSES, eval_types=['bev', '3d'])
    info = infos[0]
    for k in ('P0', 'R0_rect', 'Tr_velo_to_cam'):
        arrays[f'info_calib_{k}'] = info['calib'][k]
    arrays['info_image_shape'] = info['image']['image_shape']
    arrays['info_image_idx'] = np.array([i['image']['image_idx'] for i in infos], np.int64)
    np.savez_compressed(os.path.join(HERE, 'waymo_kitti.npz'), **arrays)
    with open(os.path.join(HERE, 'waymo_kitti.json'), 'w') as fh:
        json.dump({'classes': CLASSES, 'pcd_limit_range': PCD_LIMIT_RANGE,
                   'num_frames': NUM_FRAMES, 'submission': texts,
                   'plain': {'result_str': plain_str,
                             'ret_dict': {k: float(v) for k, v in plain.items()}},
                   'pts_bbox': {'frames': wrapped_frames, 'result_str': wrapped_str,
                                'ret_dict': {f'pts_bbox/{k}': float('{:.4f}'.format(v))
                                             for k, v in wrapped_d.items()}}}, fh, indent=1)
    print({f: len(a['name']) for f, a in enumerate(annos)}, len(texts))
    print(plain_str)


if __name__ == '__main__':
    main()
