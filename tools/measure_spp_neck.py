#!/usr/bin/env python
"""Times SPPUNetNeck at the benchmarked KITTI input (384 x 1248, one image): the C-ABI forward
with preallocated outputs, the ``modules.SPPUNetNeck`` call, and the same reference ops as eager
cuDNN (TF32 off and on).  Prints the per-kernel table of ``profile_report``, the GFLOP and
algorithmic bytes computed from the shapes, the card and its power limit, and the neck's share of
a KITTI frame (two neck calls next to ``bench.py``'s step, given with --frame-ms).  Ends with one
JSON line.  Run on an H100:

    python tools/measure_spp_neck.py [--launches 50] [--frame-ms MS]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from tests.test_spp_neck import NECK_CFG, spp_unet_neck_forward  # noqa: E402

H, W = 384, 1248


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(), 'unknown', 'unknown'
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def per_launch_ms(fn, launches, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def work(h, w):
    """(GFLOP, algorithmic MB) of one image: every conv's MACs x 2; bytes = each layer's inputs
    read once and outputs written once, fp32."""
    h2, w2, h4, w4 = h // 2, w // 2, h // 4, w // 4
    convs = [(512, 64, h4, w4, 9), (512, 128, h4, w4, 9), (128, 32, h4, w4, 9),
             (64, 64, h2, w2, 9), (64, 32, h2, w2, 9), (3, 32, h, w, 9), (32, 32, h, w, 9),
             (32, 32, h, w, 1)]
    flops = sum(2.0 * ci * co * hh * ww * k for ci, co, hh, ww, k in convs)
    floats = (3 * h * w + 64 * h2 * w2 + 3 * 128 * h4 * w4       # inputs
              + 2 * 512 * h4 * w4                                 # concat written, read by 2 convs
              + (64 + 128 + 32) * h4 * w4 * 2                     # raw outputs written + read
              + (64 + 64) * h2 * w2 * 2 + 64 * h2 * w2 * 2 + 32 * h2 * w2 * 2
              + 32 * h * w * 2                                    # x1
              + 32 * h * w * 2 + 32 * h * w + 32 * h4 * w4)       # lastconv raw, outputs
    return flops / 1e9, 4.0 * floats / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=50)
    ap.add_argument('--frame-ms', type=float, default=None,
                    help="bench.py's ms_per_step of the KITTI workload, measured in the same run")
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    feats, sd = syn.make_spp_neck_case(43, H, W)
    fc = [f.cuda().contiguous() for f in feats]
    m = modules.SPPUNetNeck(**NECK_CFG).cuda().eval()
    m.load_state_dict(sd, strict=True)
    res = dict(card=card(), shape=[H, W])
    res['gflop'], res['algorithmic_mb'] = work(H, W)
    with torch.no_grad():
        m(fc)
        torch.cuda.synchronize()
        L = capi.lib()
        cl = torch.empty((H, W, 32), device='cuda')
        nchw = torch.empty((1, 32, H, W), device='cuda')
        sem = torch.empty((1, 32, H // 4, W // 4), device='cuda')
        ptrs = [ctypes.c_void_p(t.data_ptr()) for t in fc + [cl, nchw, sem]]
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def capi_fwd():
            capi.check(L.dfm_spp_neck_forward(m._handle, *ptrs, stream), 'dfm_spp_neck_forward')
        res['capi_ms'] = per_launch_ms(capi_fwd, args.launches)
        res['module_ms'] = per_launch_ms(lambda: m(fc), args.launches)
        p = {k: v.cuda() for k, v in sd.items()}
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            res[f'cudnn_eager_{"tf32" if tf32 else "fp32"}_ms'] = per_launch_ms(
                lambda: spp_unet_neck_forward(p, fc), args.launches)
        torch.backends.cudnn.allow_tf32 = False
        # per-kernel table: one profiled call
        capi.profile_report()
        capi.profile_enable(True)
        capi_fwd()
        torch.cuda.synchronize()
        rep = capi.profile_report()
        capi.profile_enable(False)
    print(f"card: {res['card']}")
    print(f"{'kernel':60s} {'launches':>8s} {'ms':>8s} {'TFLOP/s':>8s}")
    for k, v in sorted(rep.items(), key=lambda kv: -kv[1]['ms']):
        tf = v['flops'] / (v['ms'] * 1e-3) / 1e12 if v['flops'] and v['ms'] else 0.0
        print(f"{k:60s} {v['launches']:8d} {v['ms']:8.3f} {tf:8.1f}")
    res['kernels'] = rep
    res['achieved_tflops'] = res['gflop'] / res['capi_ms']   # GFLOP / ms = TFLOP/s
    if args.frame_ms:
        res['frame_ms'] = args.frame_ms
        res['neck_share_of_frame'] = 2 * res['capi_ms'] / (2 * res['capi_ms'] + args.frame_ms)
    print(f"{res['gflop']:.1f} GFLOP, {res['algorithmic_mb']:.0f} MB per image; "
          f"C-ABI {res['capi_ms']:.3f} ms, module {res['module_ms']:.3f} ms, cuDNN eager fp32 "
          f"{res['cudnn_eager_fp32_ms']:.3f} ms, tf32 {res['cudnn_eager_tf32_ms']:.3f} ms")
    print(json.dumps(res))


if __name__ == '__main__':
    main()
