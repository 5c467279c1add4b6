#!/usr/bin/env python
"""Times MultiViewDfM's image backbone ``ResNet`` (ResNet-101 with DCNv2 in layer3 / layer4, both
Waymo configs) at 832 x 1248 for 5 and 10 images per call: the C-ABI forward with preallocated
outputs, the ``modules.ResNet`` call, and the same ops in eager PyTorch (cuDNN convs with TF32 off
and on, ``torchvision.ops.deform_conv2d`` on CUDA for the deformable convs), with CUDA events
after warm-up.  Reports algorithmic TFLOP/s on the shapes' conv FLOPs, the per-kernel split of
one profiled call (the library's event timing, a separate run), and for the deformable convs the
time an ideal MMA pipe would need for their 3 bf16 products per FLOP at the 989 TFLOP/s data-sheet
peak against the measured kernel time (the rest is gather and hand-over).  Reads the card and
its power limit in the same run.  Ends with one JSON line.  Run on an H100:

    python tools/measure_resnet101.py [--iters 10]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from tests.test_resnet101 import BACKBONE_CFG, _bn, blocks, STAGE_BLOCKS  # noqa: E402

H, W = 832, 1248
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
    """(all conv FLOPs, FLOPs of the deformable convs) of one image."""
    sizes = modules.ResNet.output_sizes(h, w)
    p = [a * b for a, b in sizes]
    total = 2 * p[0] * 147 * 64
    dcn = 0
    for name, s, j, stride, is_dcn in blocks():
        planes = 64 << s
        pin = p[s] if (j == 0 and s > 0) else p[s + 1]
        pout = p[s + 1]
        cin = (64 if s == 0 else 2 * planes) if j == 0 else 4 * planes
        total += 2 * pin * cin * planes + 2 * pout * planes * 4 * planes
        total += 2 * pout * 9 * planes * planes
        if j == 0:
            total += 2 * pout * cin * 4 * planes
        if is_dcn:
            total += 2 * pout * 9 * planes * 27
            dcn += 2 * pout * 9 * planes * planes
    return total, dcn


def eager_forward(p, img, deform_conv2d):
    """The backbone in eager PyTorch: cuDNN convs, torchvision's deformable conv."""
    x = F.max_pool2d(F.relu(_bn(F.conv2d(img, p['conv1.weight'], None, 2, 3), p, 'bn1')), 3, 2, 1)
    outs = []
    for name, s, j, stride, dcn in blocks():
        a = F.relu(_bn(F.conv2d(x, p[name + '.conv1.weight']), p, name + '.bn1'))
        if dcn:
            o = F.conv2d(a, p[name + '.conv2.conv_offset.weight'],
                         p[name + '.conv2.conv_offset.bias'], stride, 1)
            a = deform_conv2d(a, o[:, :18], p[name + '.conv2.weight'], None, stride=stride,
                              padding=1, mask=torch.sigmoid(o[:, 18:]))
        else:
            a = F.conv2d(a, p[name + '.conv2.weight'], None, stride, 1)
        a = F.relu(_bn(a, p, name + '.bn2'))
        y = _bn(F.conv2d(a, p[name + '.conv3.weight']), p, name + '.bn3')
        if j == 0:
            x = _bn(F.conv2d(x, p[name + '.downsample.0.weight'], None, stride), p,
                    name + '.downsample.1')
        x = F.relu(y + x)
        if j == STAGE_BLOCKS[s] - 1:
            outs.append(x)
    return outs


def timed(fn, iters, warm=2):
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
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    res = dict(card=card(), shape=[H, W])
    total, dcn_part = flops(H, W)
    res['gflop_per_image'] = total / 1e9
    print(res['card'], f'{total / 1e9:.1f} GFLOP per image ({dcn_part / 1e9:.1f} in the '
          'deformable convs)')
    try:
        from torchvision.ops import deform_conv2d
        deform_conv2d(torch.zeros(1, 1, 3, 3, device='cuda'), torch.zeros(1, 18, 3, 3, device='cuda'),
                      torch.zeros(1, 1, 3, 3, device='cuda'), padding=1)
    except Exception as e:   # noqa: BLE001
        deform_conv2d = None
        res['eager'] = f'torchvision.ops.deform_conv2d on CUDA is absent ({type(e).__name__})'
        print(res['eager'])
    L = capi.lib()
    for b in (5, 10):
        img, sd = syn.make_resnet101_case(71, H, W, b)
        img = img.cuda()
        m = modules.ResNet(**BACKBONE_CFG)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().eval()
        p = {k: v.cuda() for k, v in sd.items() if v.is_floating_point()}
        with torch.no_grad():
            outs = m(img)
            hd = m._handle
            arr = (ctypes.c_void_p * 4)(*[o.data_ptr() for o in outs])
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            t_c = timed(lambda: L.dfm_resnet101_forward(hd, ctypes.c_void_p(img.data_ptr()), arr,
                                                        st), args.iters)
            t_mod = timed(lambda: m(img), args.iters)
            row = dict(c_api_ms=t_c, module_ms=t_mod)
            if deform_conv2d is not None:
                for tf32 in (False, True):
                    torch.backends.cudnn.allow_tf32 = tf32
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    row[f'eager_tf32_{"on" if tf32 else "off"}_ms'] = timed(
                        lambda: eager_forward(p, img, deform_conv2d), max(2, args.iters // 2))
                torch.backends.cudnn.allow_tf32 = False
                torch.backends.cuda.matmul.allow_tf32 = False
        row['tflops_c_api'] = b * total / (t_c * 1e-3) / 1e12
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
            kind = k.split('<')[0]
            tag = ',dcn' if ',dcn' in k else ',off' if ',off' in k else ''
            shape = k.split('<')[1].split(',')[0] + ',k' + k.split(',k')[1][0] if ',k' in k else ''
            g = f'{kind}<{shape}{tag}>' if shape else kind
            a = groups.setdefault(g, dict(ms=0.0, flops=0.0, launches=0))
            a['ms'] += v['ms']
            a['flops'] += v.get('flops', 0.0)
            a['launches'] += v['launches']
        all_ms = sum(a['ms'] for a in groups.values())
        dcn_ms = sum(a['ms'] for g, a in groups.items() if ',dcn' in g)
        row['dcn_kernel_ms'] = dcn_ms
        row['dcn_mma_floor_ms'] = 3 * b * dcn_part / (BF16_TFLOPS * 1e12) * 1e3
        row['kernels'] = {g: dict(ms=round(a['ms'], 4), launches=a['launches'],
                                  share=round(a['ms'] / all_ms, 3),
                                  tflops=round(a['flops'] / (a['ms'] * 1e-3) / 1e12, 1)
                                  if a['ms'] and a['flops'] else None)
                          for g, a in sorted(groups.items(), key=lambda x: -x[1]['ms'])}
        res[f'B{b}'] = row
        print(f'B={b}: C API {t_c:.2f} ms ({row["tflops_c_api"]:.0f} TFLOP/s), module '
              f'{t_mod:.2f} ms, eager fp32 {row.get("eager_tf32_off_ms", float("nan")):.2f} ms, '
              f'eager TF32 {row.get("eager_tf32_on_ms", float("nan")):.2f} ms; deformable convs '
              f'{dcn_ms:.2f} ms against an MMA floor of {row["dcn_mma_floor_ms"]:.2f} ms')
        for g, a in row['kernels'].items():
            print(f'   {g:44s} {a["ms"]:8.3f} ms  x{a["launches"]:3d}  {100 * a["share"]:5.1f} %  '
                  f'{a["tflops"]} TFLOP/s')
        del m, outs
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
