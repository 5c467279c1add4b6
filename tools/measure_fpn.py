#!/usr/bin/env python
"""Times the Waymo image neck ``FPN`` at the shipped pyramid (input 832 x 1248: C2..C5 =
256 @ 208 x 312 .. 2048 @ 26 x 39) for N = 5 (one camsync frame) and N = 10 (the two frames of
the 10-sweep config in one call): the C-ABI forward with preallocated outputs, the
``modules.FPN`` call, and the same ops as eager cuDNN (TF32 off and on).  Prints the per-kernel
table of one profiled call, the GFLOP and compulsory HBM traffic computed from the shapes (inputs
read once, outputs written once, fp32), the share of the data-sheet HBM bandwidth, and the card
and its power limit, read in the same run.  Ends with one JSON line.  Run on an H100:

    python tools/measure_fpn.py [--launches 50]
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
from tests.test_fpn import IN_CH, fpn_forward, levels, make_inputs, make_params  # noqa: E402

H, W = 832, 1248
HBM_TBS = 3.35      # H100 SXM data sheet, HBM3


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


def work(n):
    """(GFLOP, compulsory MB) of one call on n images: lateral and fpn_conv MACs x 2; bytes =
    C2..C5 read once and the four outputs written once, fp32."""
    sizes = levels(H, W)
    flops = sum(2.0 * (c * 64 + 9 * 64 * 64) * h * w for c, (h, w) in zip(IN_CH, sizes))
    floats = sum((c + 64) * h * w for c, (h, w) in zip(IN_CH, sizes))
    return n * flops / 1e9, n * 4.0 * floats / 1e6


def measure(n, launches):
    p = make_params(7)
    xs = make_inputs(8, H, W, n, device='cuda')
    m = modules.FPN(IN_CH, 64, 4).cuda().eval()
    m.load_state_dict(p, strict=True)
    res = dict(images=n)
    res['gflop'], res['compulsory_mb'] = work(n)
    with torch.no_grad():
        outs = m(xs)
        torch.cuda.synchronize()
        L = capi.lib()
        arr = ctypes.c_void_p * 4
        ins = arr(*[x.data_ptr() for x in xs])
        ous = arr(*[o.data_ptr() for o in outs])
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def capi_fwd():
            capi.check(L.dfm_fpn_forward(m._handle, ins, ous, stream), 'dfm_fpn_forward')
        res['capi_ms'] = per_launch_ms(capi_fwd, launches)
        res['module_ms'] = per_launch_ms(lambda: m(xs), launches)
        pc = {k: v.cuda() for k, v in p.items()}
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            res[f'cudnn_eager_{"tf32" if tf32 else "fp32"}_ms'] = per_launch_ms(
                lambda: fpn_forward(pc, xs), launches)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        capi.profile_report()
        capi.profile_enable(True)
        capi_fwd()
        torch.cuda.synchronize()
        rep = capi.profile_report()
        capi.profile_enable(False)
    res['kernels'] = rep
    res['achieved_tflops'] = res['gflop'] / res['capi_ms']          # GFLOP / ms = TFLOP/s
    res['hbm_floor_ms'] = res['compulsory_mb'] / 1e3 / HBM_TBS      # GB / (TB/s) = ms
    res['share_of_hbm_peak'] = res['hbm_floor_ms'] / res['capi_ms']
    print(f"N = {n}: {'kernel':60s} {'launches':>8s} {'ms':>8s} {'TFLOP/s':>8s}")
    for k, v in sorted(rep.items(), key=lambda kv: -kv[1]['ms']):
        tf = v['flops'] / (v['ms'] * 1e-3) / 1e12 if v['flops'] and v['ms'] else 0.0
        print(f"       {k:60s} {v['launches']:8d} {v['ms']:8.3f} {tf:8.1f}")
    print(f"N = {n}: {res['gflop']:.1f} GFLOP, {res['compulsory_mb']:.0f} MB compulsory; C-ABI "
          f"{res['capi_ms']:.3f} ms ({res['share_of_hbm_peak']:.0%} of HBM peak), module "
          f"{res['module_ms']:.3f} ms, cuDNN eager fp32 {res['cudnn_eager_fp32_ms']:.3f} ms, "
          f"tf32 {res['cudnn_eager_tf32_ms']:.3f} ms")
    del xs, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    res = dict(card=card(), shape=[H, W], levels=levels(H, W))
    print(f"card: {res['card']}")
    res['runs'] = [measure(n, args.launches) for n in (5, 10)]
    print(json.dumps(res))


if __name__ == '__main__':
    main()
