"""Times kitti_eval (depth_from_motion_b200.kitti_eval) on a synthetic KITTI-val-sized set:
3769 frames, GT and detections drawn as stated in the output, 100 detections per frame (the
DfM head's max_num).  Prints end-to-end wall time (host clock around calls that end in a
device synchronise), per-stage device time (CUDA events through the library's profiler,
median / min / max over --iters profiled calls) and
the host restatement (oracle/kitti_eval_oracle.py) on a few frames, scaled per frame.

python tools/measure_kitti_eval.py [--frames 3769] [--iters 7] [--oracle-frames 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

NAMES = ('Car', 'Pedestrian', 'Cyclist', 'Van', 'Person_sitting', 'DontCare')
MIX = (0.55, 0.12, 0.06, 0.07, 0.02, 0.18)


def synthetic(frames, gt_per_frame, dt_per_frame, seed=0):
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for _ in range(frames):
        n = int(rng.integers(1, 2 * gt_per_frame))
        names = rng.choice(NAMES, n, p=MIX).astype('<U14')
        loc = np.stack([rng.uniform(-20, 20, n), rng.uniform(1, 2, n), rng.uniform(5, 60, n)], 1)
        dims = np.stack([rng.uniform(0.6, 5, n), rng.uniform(1.4, 2, n), rng.uniform(0.5, 2, n)],
                        1)
        x0, y0 = rng.uniform(0, 1100, n), rng.uniform(120, 300, n)
        bbox = np.stack([x0, y0, x0 + rng.uniform(15, 250, n), y0 + rng.uniform(15, 150, n)], 1)
        ry = rng.uniform(-np.pi, np.pi, n)
        gts.append(dict(name=names, alpha=ry.copy(), bbox=bbox, location=loc, dimensions=dims,
                        rotation_y=ry, occluded=rng.integers(0, 3, n).astype(np.float64),
                        truncated=rng.choice([0.0, 0.1, 0.3, 0.6], n)))
        m = dt_per_frame
        src = rng.integers(0, n, m)
        sig = rng.uniform(0.05, 2.0, m)[:, None]
        dts.append(dict(
            name=rng.choice(NAMES[:3], m).astype('<U14'),
            alpha=ry[src] + rng.normal(0, 0.3, m), bbox=bbox[src] + rng.normal(0, 8, (m, 4)) * sig,
            location=loc[src] + rng.normal(0, 0.5, (m, 3)) * sig,
            dimensions=dims[src] * (1 + rng.normal(0, 0.05, (m, 3))),
            rotation_y=ry[src] + rng.normal(0, 0.2, m), score=rng.uniform(0, 1, m)))
    return gts, dts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=3769)
    ap.add_argument('--gt-per-frame', type=int, default=8)
    ap.add_argument('--dt-per-frame', type=int, default=100)
    ap.add_argument('--iters', type=int, default=7)
    ap.add_argument('--oracle-frames', type=int, default=3)
    a = ap.parse_args()
    import torch
    from depth_from_motion_b200 import capi
    from depth_from_motion_b200 import kitti_eval as ke
    from oracle import kitti_eval_oracle as orc
    if not torch.cuda.is_available():
        raise SystemExit('no GPU: nothing to measure')
    gts, dts = synthetic(a.frames, a.gt_per_frame, a.dt_per_frame)
    classes = ['Car', 'Pedestrian', 'Cyclist']
    ke.kitti_eval(gts, dts, classes)   # warm-up: module load, allocations
    torch.cuda.synchronize()
    wall = []
    for _ in range(a.iters):
        t0 = time.perf_counter()
        ke.kitti_eval(gts, dts, classes)
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
    capi.profile_enable(True)
    per_stage = {}
    for _ in range(a.iters):   # CUDA events around each stage, one profiled call at a time
        capi.profile_report()
        ke.kitti_eval(gts, dts, classes)
        torch.cuda.synchronize()
        for k, v in capi.profile_report().items():
            per_stage.setdefault(k.split('@')[0], []).append(v['ms'])
    capi.profile_enable(False)
    stages = {k: {'median': round(float(np.median(v)), 3), 'min': round(min(v), 3),
                  'max': round(max(v), 3)} for k, v in per_stage.items()}
    t0 = time.perf_counter()
    orc.evaluate(gts[:a.oracle_frames], dts[:a.oracle_frames], [0, 1, 2], [0, 1, 2], True,
                 ke.MIN_OVERLAPS)
    oracle_s = time.perf_counter() - t0
    import subprocess
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        'gpu': gpu, 'frames': a.frames,
        'gt_boxes': int(sum(len(g['name']) for g in gts)),
        'gt_mix': dict(zip(NAMES, MIX)), 'dt_per_frame': a.dt_per_frame,
        'kitti_eval_ms_median': round(float(np.median(wall)), 2),
        'kitti_eval_ms_all': [round(w, 2) for w in wall],
        'device_stage_ms': stages,
        'oracle_s_per_frame': round(oracle_s / a.oracle_frames, 3),
        'oracle_frames_timed': a.oracle_frames}))


if __name__ == '__main__':
    main()
