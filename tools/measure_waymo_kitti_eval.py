"""Times WaymoDataset's KITTI metric (depth_from_motion_b200.waymo_eval.evaluate) on a synthetic
set of Waymo-val size: 39,987 frames on the FRONT camera's calibration from
tests/golden/waymo_kitti.npz, 50-300 GT LiDAR boxes per frame (Pedestrian, Cyclist, Car, Sign;
their camera annos made by bbox2result_kitti itself), and --dt-per-frame detections per frame
jittered from the frame's GT, shaped as MultiViewDfM.simple_test returns them (CPU tensors,
labels in the configs' class order: 0 Pedestrian, 1 Cyclist, 2 Car).

For each detection count it prints the end-to-end time of evaluate (plain results: bbox, BEV,
3-D and AOS; and results wrapped as {'pts_bbox': ...} on GT without alphas: BEV and 3-D), the
time of its steps (device conversion with the gather of the evaluator rows, GT concatenation,
packing, the evaluator), the evaluator's device workspace, and the device time of each kernel
class (CUDA events through the library's profiler) of one profiled call.  Every time is a host
clock around work that ends in a device synchronise.

python tools/measure_waymo_kitti_eval.py [--frames 39987] [--dt-per-frame 100 500]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
GT_NAMES = ['Pedestrian', 'Cyclist', 'Car', 'Sign']


def lidar_boxes(rng, n, labels):
    size = np.array([(0.9, 0.9, 1.8), (1.8, 0.8, 1.7), (4.5, 2.0, 1.7), (0.3, 0.8, 0.8)])
    xyz = np.stack([rng.uniform(3, 80, n), rng.uniform(-40, 40, n), rng.uniform(-2.5, 0.5, n)],
                   1)
    dims = size[labels] * rng.uniform(0.8, 1.2, (n, 3))
    return np.concatenate([xyz, dims, rng.uniform(-np.pi, np.pi, (n, 1))], 1)


def make_set(frames, dt_per_frame, seed=0):
    import torch
    from depth_from_motion_b200 import waymo_eval as we
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'waymo_kitti.npz'))
    calib = {k: z[f'info_calib_{k}'] for k in ('P0', 'R0_rect', 'Tr_velo_to_cam')}
    infos = [{'calib': calib, 'image': {'image_shape': z['info_image_shape'],
                                        'image_idx': 1000000 + f}} for f in range(frames)]
    rng = np.random.default_rng(seed)
    ng = rng.integers(50, 301, frames)
    G = int(ng.sum())
    g_lab = rng.choice(4, G, p=(0.3, 0.1, 0.5, 0.1))
    g_box = lidar_boxes(rng, G, g_lab).astype(np.float32)
    split = lambda a, n: torch.from_numpy(a).split(list(n))
    gt_res = [dict(boxes_3d=b, scores_3d=s, labels_3d=l) for b, s, l in zip(
        split(g_box, ng), split(np.ones(G, np.float32), ng), split(g_lab, ng))]
    gts = we.bbox2result_kitti(gt_res, infos, GT_NAMES)
    for g in gts:
        n = len(g['name'])
        g['occluded'] = rng.integers(0, 3, n)
        g['truncated'] = rng.choice([0.0, 0.2, 0.4], n)
        for k in ('alpha', 'bbox', 'dimensions', 'location', 'rotation_y'):
            g[k] = g[k].astype(np.float64)
        del g['score'], g['sample_idx']
    for i, g in zip(infos, gts):
        i['annos'] = i['cam_sync_annos'] = g   # the FRONT camera's annos stand for both
    g_off = np.concatenate([[0], np.cumsum(ng)])
    D = frames * dt_per_frame
    fr = np.repeat(np.arange(frames), dt_per_frame)
    src = g_off[fr] + rng.integers(0, ng[fr])
    sig = rng.uniform(0.02, 0.6, (D, 1))
    d_box = (g_box[src] + rng.normal(0, 1, (D, 7)) * sig * [1, 1, 0.3, 0.3, 0.3, 0.3, 1]
             ).astype(np.float32)
    d_lab = np.where(g_lab[src] < 3, g_lab[src], rng.integers(0, 3, D))
    nd = np.full(frames, dt_per_frame)
    results = [dict(boxes_3d=b, scores_3d=s, labels_3d=l) for b, s, l in zip(
        split(d_box, nd), split(rng.uniform(0, 1, D).astype(np.float32), nd),
        split(d_lab, nd))]
    return results, infos, G, D


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=39987)
    ap.add_argument('--dt-per-frame', type=int, nargs='+', default=[100, 500])
    ap.add_argument('--out', default=None, help='also write the JSON here')
    a = ap.parse_args()
    import torch
    from depth_from_motion_b200 import capi
    from depth_from_motion_b200 import kitti_eval as ke
    from depth_from_motion_b200 import waymo_eval as we
    if not torch.cuda.is_available():
        raise SystemExit('no GPU: nothing to measure')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    report = {'gpu': gpu, 'frames': a.frames, 'runs': []}
    for ndt in a.dt_per_frame:
        (results, infos, G, D), t_make = timed(lambda: make_set(a.frames, ndt))
        run = {'dt_per_frame': ndt, 'gt_boxes': G, 'detections': D,
               'make_set_s': round(t_make, 2)}
        # the steps of the plain path, one by one
        gt, t = timed(lambda: ke.concat_annos(we.gt_annos_of(infos), ('name',) + ke.GT_COLS))
        run['concat_gt_s'] = round(t, 3)
        (dt, flags, rows), t = timed(lambda: we._detections(
            results, infos, we.WAYMO_CLASSES, we.WAYMO_PCD_LIMIT_RANGE, gt, None))
        run['convert_and_gather_s'] = round(t, 3)
        packed, t = timed(lambda: ke.pack_columns(gt, dt, flags, rows))
        run['pack_columns_s'] = round(t, 3)
        run['kept_detections'] = int(dt['off'][-1])
        run['pairs'] = int(packed['pair_off'][-1])
        ev = ke.KittiEvaluator([1, 2, 0], [0, 1, 2], True)
        _, t = timed(lambda: ev.forward(packed))
        ws, ov, parts = ev.workspace()
        ev.close()
        run['evaluator_s'] = round(t, 2)
        run['evaluator_workspace_gb'] = round(ws / 2**30, 2)
        run['overlap_buffer_gb'] = round(ov / 2**30, 2)
        run['parts'] = parts
        del packed, rows, dt
        # end to end, profiler off
        (ap_plain, _), t = timed(lambda: we.evaluate(results, infos, return_str=True))
        run['evaluate_plain_s'] = round(t, 2)
        run['plain_Car_3D_AP40_moderate_strict'] = ap_plain['KITTI/Car_3D_AP40_moderate_strict']
        # device time per kernel class of one profiled plain call
        capi.profile_enable(True)
        capi.profile_report()
        we.evaluate(results, infos)
        torch.cuda.synchronize()
        prof = capi.profile_report()
        capi.profile_enable(False)
        for i in infos:
            i['cam_sync_annos']['alpha'] = np.full(len(i['cam_sync_annos']['alpha']), -10.0)
        wrapped = [{'pts_bbox': r} for r in results]
        ap_w, t = timed(lambda: we.evaluate(wrapped, infos))
        run['evaluate_pts_bbox_s'] = round(t, 2)
        stages = {}
        for k, v in prof.items():
            name = k.split('@')[0]
            s = stages.setdefault(name, {'launches': 0, 'ms': 0.0})
            s['launches'] += v['launches']
            s['ms'] = round(s['ms'] + v['ms'], 2)
        run['device_ms'] = stages
        # torch's allocations only: the evaluator's workspace is its own (above)
        run['peak_torch_mem_gb'] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
        report['runs'].append(run)
        print(json.dumps(run), flush=True)
        del results, infos, wrapped
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    print(json.dumps(report))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
