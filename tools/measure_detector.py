"""Times the whole detectors' ``simple_test`` on synthetic decoded images, and ``dfm_image_prep``
against its HBM floor and against the cv2 / numpy restatement on the same host.

    python tools/measure_detector.py [--iters 20] [--warmup 3]

Workloads: KITTI 375 x 1242 pair (DfM); Waymo 5 x 1280 x 1920 (camsync); Waymo 10 x 1280 x 1920
(10 sweeps) at B = 1 and 2.  Weights are random (timing does not depend on their values; the box
count does, and the random heads fill max_num).  The per-module shares come from the library's
event profile in a separate, profiled run.  Every line ends with the card name and power
limit it was measured on.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import capi, image_prep, modules, pipeline_meta, registry  # noqa
from depth_from_motion_b200 import synthetic as syn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
CONFIGS = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'detector_configs.json')))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def detector(name, seed=0):
    det = registry.build_detector(CONFIGS[name])
    rng = np.random.RandomState(seed)
    state = {}
    for k, v in det.state_dict().items():
        if k.endswith('num_batches_tracked'):
            state[k] = v
        elif k.endswith('running_var') or v.dim() == 1 and not k.endswith('bias') and \
                not k.endswith('running_mean'):
            state[k] = torch.from_numpy((1 + 0.1 * np.abs(rng.standard_normal(v.shape)))
                                        .astype(np.float32))
        elif v.dim() <= 1:
            state[k] = torch.from_numpy((0.1 * rng.standard_normal(v.shape)).astype(np.float32))
        else:
            state[k] = torch.from_numpy((rng.standard_normal(v.shape) /
                                         np.sqrt(np.prod(v.shape[1:]))).astype(np.float32))
    det.load_state_dict(state, strict=True)
    return det.cuda().eval()


def workloads():
    rng = np.random.RandomState(1)

    def views(n, h, w):
        return [torch.from_numpy(rng.randint(0, 256, (h, w, 3), dtype=np.uint8)).cuda()
                for _ in range(n)]
    kitti = views(2, 375, 1242)
    ori = lambda t: np.diag([1 / 0.65, 1 / 0.65, 1, 1]) @ syn.waymo_lidar2img(t)  # noqa: E731

    def run_kitti():
        return image_prep.prepare_kitti(kitti[0], kitti[1:], syn.KITTI_P2,
                                        syn.KITTI_CUR2PREV[2:3])
    w5, w10a, w10b = views(5, 1280, 1920), views(10, 1280, 1920), views(10, 1280, 1920)

    def run_w(vs_list, t):
        def f():
            imgs, metas = [], []
            for vs in vs_list:
                img, m = image_prep.prepare_waymo(vs, ori(t), num_ref_frames=t - 1)
                imgs.append(img)
                metas += m
            return torch.cat(imgs), metas
        return f
    return [('KITTI 375x1242 pair', 'dfm_r34_1x8_kitti-3d-3class.py', run_kitti),
            ('Waymo 5x1280x1920', 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py',
             run_w([w5], 1)),
            ('Waymo 10x1280x1920 B=1',
             'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py',
             run_w([w10a], 2)),
            ('Waymo 10x1280x1920 B=2',
             'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py',
             run_w([w10a, w10b], 2))]


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def image_prep_row(src, mode, out_hw, crop, to_rgb, iters, gpu):
    n, h, w, _ = src.shape
    out = image_prep.image_prep(src, mode, out_hw, crop, 32, to_rgb=to_rgb)
    ms = time_ms(lambda: image_prep.image_prep(src, mode, out_hw, crop, 32, to_rgb=to_rgb),
                 iters * 5, 5)
    nbytes = src.numel() + out.numel() * 4
    floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
    host_ms = 'not measured (no cv2)'
    try:
        import cv2
        imgs = src.cpu().numpy()
        mean = np.array(image_prep.IMG_NORM_MEAN, dtype=np.float32)   # as Normalize stores them
        std = np.array(image_prep.IMG_NORM_STD, dtype=np.float32)

        def cpu():
            for v in imgs:
                if mode == 'crop':
                    v = v[crop[1]:crop[1] + out_hw[0], crop[0]:crop[0] + out_hw[1]]
                else:
                    v = cv2.resize(v.astype(np.float32), (out_hw[1], out_hw[0]),
                                   interpolation=cv2.INTER_LINEAR)
                v = v.astype(np.float32)
                if to_rgb:
                    cv2.cvtColor(v, cv2.COLOR_BGR2RGB, v)
                cv2.subtract(v, np.float64(mean.reshape(1, -1)), v)
                cv2.multiply(v, 1 / np.float64(std.reshape(1, -1)), v)
                ph, pw = -(-v.shape[0] // 32) * 32, -(-v.shape[1] // 32) * 32
                cv2.copyMakeBorder(v, 0, ph - v.shape[0], 0, pw - v.shape[1],
                                   cv2.BORDER_CONSTANT, value=0)
        cpu()
        t = time.perf_counter()
        for _ in range(3):
            cpu()
        host_ms = f'{(time.perf_counter() - t) / 3 * 1e3:.1f} ms on {os.cpu_count()} host cores'
    except ImportError:
        pass
    print(f'  dfm_image_prep {mode:7s} {n:2d} x {h}x{w} -> {tuple(out.shape)}: {ms:.3f} ms, '
          f'{nbytes / 1e6:.1f} MB compulsory, HBM floor {floor_ms:.3f} ms '
          f'({floor_ms / ms:.0%} of floor speed); cv2/numpy: {host_ms} [{gpu}]')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'measure_detector needs a GPU'
    gpu = card()
    print('image preparation:')
    rng = np.random.RandomState(2)
    k = torch.from_numpy(rng.randint(0, 256, (2, 375, 1242, 3), dtype=np.uint8)).cuda()
    x1, y1 = pipeline_meta.random_crop_offsets((375, 1242), (320, 1280), (1, 1), (0.5, 0.5))
    image_prep_row(k, 'crop', (320, 1242), (x1, y1), False, args.iters, gpu)
    for n in (5, 10):
        wv = torch.from_numpy(rng.randint(0, 256, (n, 1280, 1920, 3), dtype=np.uint8)).cuda()
        image_prep_row(wv, 'rescale', (832, 1248), (0, 0), True, args.iters, gpu)
    print('simple_test (image_prep + detector), CUDA events:')
    for label, cfg, make in workloads():
        det = detector(cfg)
        with torch.no_grad():
            ms = time_ms(lambda: det.simple_test(*make()), args.iters, args.warmup)
            capi.profile_enable(True)
            capi.profile_report()
            det.simple_test(*make())
            torch.cuda.synchronize()
            prof = capi.profile_report()
            capi.profile_enable(False)
        total = sum(v['ms'] for v in prof.values()) or 1.0
        groups = {}
        for cls, v in prof.items():
            key = cls.split('<')[0]
            groups[key] = groups.get(key, 0.0) + v['ms']
        top = sorted(groups.items(), key=lambda kv: -kv[1])[:8]
        print(f'  {label}: {ms:.2f} ms per call; profiled kernels {total:.2f} ms: ' +
              ', '.join(f'{k} {v / total:.0%}' for k, v in top) + f' [{gpu}]')
        del det
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
