#!/usr/bin/env python
"""Times DfM's image backbone ``LIGAResNet`` (KITTI config) at 384 x 1248 for B = 1 and B = 2
(cur + prev of a frame in one call): the C-ABI forward with preallocated outputs, the
``modules.LIGAResNet`` call, and the same ops as eager cuDNN (TF32 off and on), with CUDA events
after warm-up.  Reports algorithmic TFLOP/s on the shapes' conv FLOPs, the share of the 989
TFLOP/s bf16 data-sheet peak counting 3 MMAs per product for the tensor-core convs, the per-kernel
split of one profiled call (the library's event timing, a separate run) and the card and its
power limit, read in the same run.  Ends with one JSON line.  Run on an H100:

    python tools/measure_liga_resnet.py [--iters 20]
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
from tests.test_liga_resnet import BACKBONE_CFG, liga_resnet_forward  # noqa: E402

H, W = 384, 1248
BF16_TFLOPS = 989.0   # H100 SXM data sheet, dense


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(), 'unknown', 'unknown'
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def flops(h, w):
    """(all conv FLOPs, FLOPs of the 3x3 stride-1 convs) of one image."""
    (h2, w2), (h4, w4) = modules.LIGAResNet.output_sizes(h, w)
    p2, p4 = h2 * w2, h4 * w4
    stem = 2 * p2 * 147 * 64
    l1 = 6 * 2 * p2 * 576 * 64
    s2 = 2 * p4 * 576 * 128 + 2 * p4 * 64 * 128
    s1 = 25 * 2 * p4 * 1152 * 128
    return stem + l1 + s2 + s1, l1 + s1


def timed(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    res = dict(card=card(), shape=[H, W])
    total, tc_part = flops(H, W)
    res['gflop_per_image'] = total / 1e9
    print(res['card'], f'{total / 1e9:.1f} GFLOP per image ({tc_part / 1e9:.1f} in 3x3 stride-1)')
    L = capi.lib()
    for b in (1, 2):
        img, sd = syn.make_liga_resnet_case(71, H, W, b)
        img = img.cuda()
        m = modules.LIGAResNet(**BACKBONE_CFG)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().eval()
        p = {k: v.cuda() for k, v in sd.items() if v.is_floating_point()}
        with torch.no_grad():
            outs = m(img)
            hd = m._handle
            arr = (ctypes.c_void_p * 4)(*[o.data_ptr() for o in outs])
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            t_c = timed(lambda: L.dfm_liga_resnet_forward(hd, ctypes.c_void_p(img.data_ptr()), arr,
                                                          st), args.iters)
            t_mod = timed(lambda: m(img), args.iters)
            row = dict(c_api_ms=t_c, module_ms=t_mod)
            for tf32 in (False, True):
                torch.backends.cudnn.allow_tf32 = tf32
                torch.backends.cuda.matmul.allow_tf32 = tf32
                row[f'cudnn_tf32_{"on" if tf32 else "off"}_ms'] = timed(
                    lambda: liga_resnet_forward(p, img), args.iters)
            torch.backends.cudnn.allow_tf32 = False
        row['tflops_c_api'] = b * total / (t_c * 1e-3) / 1e12
        row['tflops_cudnn_fp32'] = b * total / (row['cudnn_tf32_off_ms'] * 1e-3) / 1e12
        # per-kernel split of one profiled call (separate run)
        with torch.no_grad():
            capi.profile_report()
            capi.profile_enable(True)
            m(img)
            capi.sync_check()
            rep = capi.profile_report()
            capi.profile_enable(False)
        groups = {}
        for k, v in rep.items():
            g = k.split('<')[0] + ('<' + k.split('<')[1].split(',')[0] + (
                ',' + k.split(',d')[-1].split('>')[0] if 'conv_tc' in k else '') if '<' in k else '')
            a = groups.setdefault(g, dict(ms=0.0, flops=0.0, launches=0))
            a['ms'] += v['ms']
            a['flops'] += v.get('flops', 0.0)
            a['launches'] += v['launches']
        tc_ms = sum(a['ms'] for g, a in groups.items() if g.startswith('resnet_conv_tc'))
        all_ms = sum(a['ms'] for a in groups.values())
        row['tc_kernel_ms'] = tc_ms
        row['tc_tflops'] = b * tc_part / (tc_ms * 1e-3) / 1e12 if tc_ms else 0.0
        row['tc_share_of_bf16_peak_3mma'] = 3 * row['tc_tflops'] / BF16_TFLOPS
        row['kernels'] = {g: dict(ms=round(a['ms'], 4), launches=a['launches'],
                                  share=round(a['ms'] / all_ms, 3),
                                  tflops=round(a['flops'] / (a['ms'] * 1e-3) / 1e12, 1)
                                  if a['ms'] and a['flops'] else None)
                          for g, a in sorted(groups.items(), key=lambda x: -x[1]['ms'])}
        res[f'B{b}'] = row
        print(f'B={b}: C API {t_c:.3f} ms ({row["tflops_c_api"]:.0f} TFLOP/s), module '
              f'{t_mod:.3f} ms, cuDNN fp32 {row["cudnn_tf32_off_ms"]:.3f} ms, cuDNN TF32 '
              f'{row["cudnn_tf32_on_ms"]:.3f} ms; tensor-core convs {tc_ms:.3f} ms = '
              f'{row["tc_tflops"]:.0f} TFLOP/s ({100 * row["tc_share_of_bf16_peak_3mma"]:.0f} % of '
              'the bf16 peak at 3 MMAs per product)')
        for g, a in row['kernels'].items():
            print(f'   {g:40s} {a["ms"]:8.3f} ms  x{a["launches"]:3d}  {100 * a["share"]:5.1f} %  '
                  f'{a["tflops"]} TFLOP/s')
        del m, outs
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
