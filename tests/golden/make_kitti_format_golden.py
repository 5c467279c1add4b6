"""Writes tests/golden/kitti_format.npz + kitti_format.json: KittiDataset.convert_valid_bboxes
and KittiDataset.bbox2result_kitti of mmdet3d (datasets/kitti_dataset.py), the two methods'
source executed verbatim through oracle/ref_loader with the reference's own
LiDARInstance3DBoxes / Box3DMode / points_cam2img (core/bbox/structures).  mmcv.ops, which
the box structures import but these methods never call, is stubbed.

Also stored: the demo frame's data_info (calibration, image shape, GT annos), so the tests
can rebuild data_infos without the reference tree.

Input: 6 frames of LiDAR boxes around the demo frame's calibration
(demo/data/kitti/kitti_000008_infos.pkl, image_idx changed per frame), some inside and some
outside the image and the point-cloud range, yaws past +-pi, and one empty frame.  Output per
frame and for pseudo_lidar False / True: every array of the KITTI-format anno and the text of
the submission file.

Run from the repository root: python tests/golden/make_kitti_format_golden.py
"""
import ast
import copy
import json
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from oracle import ref_loader as rl  # noqa: E402

KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
        'rotation_y', 'score', 'sample_idx')
CLASSES = ['Pedestrian', 'Cyclist', 'Car']
PCD_LIMIT_RANGE = [0, -40, -3, 70.4, 40, 0.0]


def load_structures():
    rl.load_reference()
    for n in ('mmcv', 'mmdet3d', 'mmdet3d.core', 'mmdet3d.core.utils', 'mmdet3d.core.bbox',
              'mmdet3d.core.bbox.structures'):
        if n not in sys.modules:
            rl._pkg(n)
    if 'mmdet3d.core.bbox.structures.utils' not in sys.modules:
        ac = rl._exec('mmdet3d.core.utils.array_converter', 'mmdet3d/core/utils/array_converter.py')
        sys.modules['mmdet3d.core.utils'].array_converter = ac.array_converter
        rl._exec('mmdet3d.core.bbox.structures.utils', 'mmdet3d/core/bbox/structures/utils.py')
    ops = rl._pkg('mmcv.ops')
    for n in ('box_iou_rotated', 'points_in_boxes_all', 'points_in_boxes_part'):
        setattr(ops, n, None)
    sys.modules['mmcv'].ops = ops
    pts = rl._pkg('mmdet3d.core.points')
    pts.BasePoints = type('BasePoints', (), {})
    S = 'mmdet3d/core/bbox/structures/'
    mods = {m: rl._exec('mmdet3d.core.bbox.structures.' + m, S + m + '.py')
            for m in ('base_box3d', 'cam_box3d', 'depth_box3d', 'lidar_box3d', 'box_3d_mode')}
    return (mods['lidar_box3d'].LiDARInstance3DBoxes, mods['box_3d_mode'].Box3DMode,
            sys.modules['mmdet3d.core.bbox.structures.utils'].points_cam2img)


def dataset_methods(namespace):
    """KittiDataset.convert_valid_bboxes / bbox2result_kitti, their source unchanged."""
    path = os.path.join(rl.REFERENCE_ROOT, 'mmdet3d/datasets/kitti_dataset.py')
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body
               if isinstance(n, ast.ClassDef) and n.name == 'KittiDataset')
    out = {}
    for fn in cls.body:
        if isinstance(fn, ast.FunctionDef) and fn.name in ('convert_valid_bboxes',
                                                          'bbox2result_kitti'):
            code = ast.get_source_segment(src, fn)
            code = '\n'.join(l[4:] if l.startswith('    ') else l for l in code.split('\n'))
            exec(compile(code, path, 'exec'), namespace)
            out[fn.name] = namespace[fn.name]
    return out


class _Mmcv:
    @staticmethod
    def mkdir_or_exist(p):
        os.makedirs(p, exist_ok=True)

    @staticmethod
    def track_iter_progress(x):
        return x


def make_inputs(seed=0):
    with open(os.path.join(rl.REFERENCE_ROOT, 'demo/data/kitti/kitti_000008_infos.pkl'),
              'rb') as f:
        info = pickle.load(f)[0]
    rng = np.random.default_rng(seed)
    infos, results = [], []
    for f in range(6):
        i = copy.deepcopy(info)
        i['image']['image_idx'] = 8 + f
        infos.append(i)
        n = 0 if f == 3 else int(rng.integers(4, 12))
        x = rng.uniform(-5, 75, n)          # part outside the 0..70.4 range
        y = rng.uniform(-30, 30, n)
        z = rng.uniform(-2.5, 0.5, n)
        dims = np.stack([rng.uniform(0.5, 4.5, n), rng.uniform(0.5, 2, n),
                         rng.uniform(1.2, 2, n)], 1)
        yaw = rng.uniform(-4, 4, n)         # limit_yaw folds these into [-pi, pi)
        boxes = np.concatenate([np.stack([x, y, z], 1), dims, yaw[:, None]], 1)
        results.append(dict(boxes_3d=torch.tensor(boxes, dtype=torch.float32),
                            scores_3d=torch.tensor(rng.uniform(0, 1, n), dtype=torch.float32),
                            labels_3d=torch.tensor(rng.integers(0, 3, n))))
    return infos, results


def main():
    LiDARBoxes, Box3DMode, points_cam2img = load_structures()
    ns = dict(np=np, torch=torch, mmcv=_Mmcv, Box3DMode=Box3DMode,
              points_cam2img=points_cam2img)
    methods = dataset_methods(ns)
    infos, results = make_inputs()
    arrays, texts = {}, {}
    for f, r in enumerate(results):
        arrays[f'in{f}_boxes_3d'] = r['boxes_3d'].numpy()
        arrays[f'in{f}_scores_3d'] = r['scores_3d'].numpy()
        arrays[f'in{f}_labels_3d'] = r['labels_3d'].numpy()
    for pseudo in (False, True):
        ds = type('Dataset', (), {})()
        ds.pseudo_lidar, ds.pcd_limit_range, ds.data_infos = pseudo, PCD_LIMIT_RANGE, infos
        ds.convert_valid_bboxes = methods['convert_valid_bboxes'].__get__(ds)
        wrapped = [dict(boxes_3d=LiDARBoxes(r['boxes_3d'].clone()),
                        scores_3d=r['scores_3d'], labels_3d=r['labels_3d']) for r in results]
        with tempfile.TemporaryDirectory() as tmp:
            annos = methods['bbox2result_kitti'](ds, wrapped, CLASSES, None, tmp)
            for i in infos:
                idx = i['image']['image_idx']
                with open(f'{tmp}/{idx:06d}.txt') as fh:
                    texts[f'{int(pseudo)}_{idx:06d}'] = fh.read()
        for f, a in enumerate(annos):
            for k in KEYS:
                arrays[f'out{int(pseudo)}_{f}_{k}'] = np.asarray(a[k])
    # the demo frame's data_info: calibration, image and GT annos (image_idx 8 + frame)
    info = infos[0]
    for k in ('P2', 'R0_rect', 'Tr_velo_to_cam'):
        arrays[f'info_calib_{k}'] = info['calib'][k]
    arrays['info_image_shape'] = info['image']['image_shape']
    for k in ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
              'rotation_y', 'score', 'difficulty'):
        arrays[f'info_annos_{k}'] = info['annos'][k]
    np.savez_compressed(os.path.join(HERE, 'kitti_format.npz'), **arrays)
    with open(os.path.join(HERE, 'kitti_format.json'), 'w') as fh:
        json.dump({'classes': CLASSES, 'pcd_limit_range': PCD_LIMIT_RANGE,
                   'submission': texts}, fh, indent=1)
    print({k: len(v.splitlines()) for k, v in texts.items()})


if __name__ == '__main__':
    main()
