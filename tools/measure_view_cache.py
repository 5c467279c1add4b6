"""Times ``simple_test`` on video with the per-view feature cache off and on, and the cache's two
kernels against HBM bandwidth.

    python tools/measure_view_cache.py [--iters 20] [--rounds 2]

Workloads (synthetic uint8 images already on the device, random weights as in
measure_detector.py; each timed call is ``prepare_*`` + ``simple_test``, CUDA events over
``--iters`` calls after warm-up):
  KITTI t-1       DfM, each call's previous frame is the last call's current frame
  Waymo t-10      MultiViewDfM 10 sweeps, reference frame ten calls back (max_views 100)
  Waymo t-1       MultiViewDfM 10 sweeps, reference frame one call back (max_views 10)
Each is run with the cache off, on, and on with every reference frame new (all miss: the
KITTI-3D evaluation case, where consecutive samples are not consecutive frames).  Off and on
alternate for ``--rounds`` rounds in one process.  Every line ends with the card name and power
limit it was measured on.
"""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from depth_from_motion_b200 import capi, image_prep, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from measure_detector import HBM_BYTES_PER_S, card, detector  # noqa: E402

KITTI = 'dfm_r34_1x8_kitti-3d-3class.py'
SWEEPS10 = 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py'


def frames(n, h, w, views, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return [[torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda', generator=g)
             for _ in range(views)] for _ in range(n)]


def time_calls(det, make, ts):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for t in ts:
        det.simple_test(*make(t))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / len(ts)


def workload(label, det, make_seq, make_fresh, lag, cap, iters, rounds, gpu):
    """make_seq(t): the call at time t of a video whose reference frame is t - lag;
    make_fresh(t): the same current frame with a reference frame no call has seen."""
    warm = lag + 3
    ts = range(warm, warm + iters)
    rows = {'off': [], 'on': [], 'all-miss': []}
    with torch.no_grad():
        for _ in range(rounds):
            det.set_feature_cache(0)
            for t in range(warm):
                det.simple_test(*make_seq(t))
            rows['off'].append(time_calls(det, make_seq, ts))
            det.set_feature_cache(cap)
            for t in range(warm):
                det.simple_test(*make_seq(t))
            rows['on'].append(time_calls(det, make_seq, ts))
            st = det.feature_cache_stats()
            det.set_feature_cache(cap)
            for t in range(warm):
                det.simple_test(*make_fresh(t))
            rows['all-miss'].append(time_calls(det, make_fresh, ts))
            st_miss = det.feature_cache_stats()
    det.set_feature_cache(0)
    off, on, miss = (float(np.median(rows[k])) for k in ('off', 'on', 'all-miss'))
    print(f'  {label}: off {off:.2f} ms, on {on:.2f} ms ({off - on:+.2f} ms saved, '
          f'{(off - on) / off:.1%}), all-miss {miss:.2f} ms ({miss - off:+.2f} ms, '
          f'{(miss - off) / off:+.2%}); per round off {rows["off"]}, on {rows["on"]}, '
          f'all-miss {rows["all-miss"]}; cache after the hit run: {st}; after the all-miss '
          f'run: {st_miss} [{gpu}]', flush=True)


def kernel_rates(gpu):
    L = capi.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for label, n, shape in (('KITTI pair', 2, (3, 320, 1248)),
                            ('Waymo 10 views', 10, (3, 832, 1248))):
        x = torch.randn((n,) + shape, device='cuda')
        y = x.clone()
        out = torch.empty((n, 2), dtype=torch.int64, device='cuda')
        mism = torch.empty(n, dtype=torch.int32, device='cuda')
        elems = x[0].numel()
        a = (ctypes.c_void_p * n)(*[x[i].data_ptr() for i in range(n)])
        b = (ctypes.c_void_p * n)(*[y[i].data_ptr() for i in range(n)])
        for name, fn, nbytes in (
                ('dfm_view_fingerprint', lambda: L.dfm_view_fingerprint(
                    ctypes.c_void_p(x.data_ptr()), n, elems, ctypes.c_void_p(out.data_ptr()),
                    st), x.numel() * 4),
                ('dfm_views_equal', lambda: L.dfm_views_equal(
                    a, b, n, elems, ctypes.c_void_p(mism.data_ptr()), st), 2 * x.numel() * 4)):
            for _ in range(5):
                fn()
            reps = 200
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            print(f'  {name} {label} ({nbytes / 1e6:.1f} MB read): {ms * 1e3:.1f} us, '
                  f'{nbytes / ms / 1e6:.0f} GB/s = {nbytes / ms / 1e-3 / HBM_BYTES_PER_S:.0%} '
                  f'of 3.35 TB/s [{gpu}]', flush=True)
        capi.sync_check()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'measure_view_cache needs a GPU'
    gpu = card()
    print('cache kernels (CUDA events over 200 launches, memset included):')
    kernel_rates(gpu)
    print('prepare + simple_test per call, CUDA events:')
    n = 10 + 3 + args.iters

    det = detector(KITTI)
    kf = [f[0] for f in frames(n, 375, 1242, 1, 1)]
    kfresh = [f[0] for f in frames(n, 375, 1242, 1, 2)]

    def kitti(cur, prev):
        return image_prep.prepare_kitti(cur, [prev], syn.KITTI_P2, syn.KITTI_CUR2PREV[2:3])
    workload('KITTI t-1', det, lambda t: kitti(kf[t + 1], kf[t]),
             lambda t: kitti(kf[t + 1], kfresh[t]), 1, 2, args.iters, args.rounds, gpu)
    del det
    torch.cuda.empty_cache()

    det = detector(SWEEPS10)
    wf = frames(n, 1280, 1920, 5, 3)
    wfresh = frames(n, 1280, 1920, 5, 4)
    ori = np.diag([1 / 0.65, 1 / 0.65, 1, 1]) @ syn.waymo_lidar2img(2)

    def waymo(cur, ref):
        return image_prep.prepare_waymo(cur + ref, ori, num_ref_frames=1)
    for lag, cap in ((10, 100), (1, 10)):
        workload(f'Waymo 10-sweep t-{lag}', det,
                 lambda t, lag=lag: waymo(wf[t], wf[max(t - lag, 0)]),
                 lambda t: waymo(wf[t], wfresh[t]), lag, cap, args.iters, args.rounds, gpu)
    capi.sync_check()


if __name__ == '__main__':
    main()
