#!/usr/bin/env python
"""Times Anchor3DHead's forward (the 1x1-conv tensor-core GEMM of csrc/head1x1_tc.cuh) at the
shipped Waymo shape, [1, 256, 300, 220] -> 18 + 42 + 12 channels, against the same three convs
as F.conv2d (cuDNN, TF32 off and on), and its share of a whole Waymo sample (lifting + neck +
head against lifting + neck, the bench.py waymo_mv / waymo_10sweep paths).  Prints the card and
its power limit, then one JSON line.  Run on an H100:

    python tools/measure_anchor3d_head.py [--launches 200]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402

FEAT, NY, NX = 256, 300, 220
ROWS = (18, 42, 12)                   # cls, reg, dir
HBM_BYTES = 4 * NY * NX * (FEAT + sum(ROWS))   # read the map once, write the three outputs
HBM_PEAK = 3.35e12                    # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(), 'unknown', 'unknown'
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def per_launch_ms(fn, launches, warmup=20):
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


def head_module(rng):
    m = modules.Anchor3DHead(
        num_classes=3, in_channels=FEAT, feat_channels=FEAT,
        anchor_generator=dict(type='AlignedAnchor3DRangeGenerator',
                              sizes=[[0.91, 0.84, 1.74], [1.81, 0.84, 1.77],
                                     [4.73, 2.08, 1.77]], rotations=[0, 1.57]))
    sd = {k: torch.from_numpy((rng.standard_normal(v.shape) / 16).astype(np.float32))
          for k, v in m.state_dict().items()}
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), {k: v.cuda() for k, v in sd.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    out = dict(card=card())
    rng = np.random.RandomState(0)
    head, sd = head_module(rng)
    x = torch.from_numpy(np.maximum(rng.standard_normal((1, FEAT, NY, NX)), 0)
                         .astype(np.float32)).cuda()
    res = {}
    with torch.no_grad():
        head([x])                         # builds the handle and uploads the weights
        capi.sync_check()
        # the kernel alone: the C entry point on preallocated outputs
        L = capi.lib()
        bufs = [torch.empty((c, NY, NX), device='cuda') for c in ROWS]
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        args_c = [head._handle, ctypes.c_void_p(x.data_ptr())] + \
                 [ctypes.c_void_p(b.data_ptr()) for b in (bufs[0], bufs[1], bufs[2])] + [stream]

        def raw():
            L.dfm_anchor3d_head_forward(*args_c)
        ms = per_launch_ms(raw, args.launches)
        capi.sync_check()
        res['head1x1_tc'] = dict(ms=round(ms, 4), gbs=round(HBM_BYTES / ms / 1e6, 1),
                                 hbm_fraction=round(HBM_BYTES / (ms * 1e-3) / HBM_PEAK, 3))
        ms = per_launch_ms(lambda: head([x]), args.launches)
        res['Anchor3DHead_module_call'] = dict(ms=round(ms, 4))
        # the three convs as F.conv2d (cuDNN)
        w = [sd[k + '.weight'] for k in ('conv_cls', 'conv_reg', 'conv_dir_cls')]
        b = [sd[k + '.bias'] for k in ('conv_cls', 'conv_reg', 'conv_dir_cls')]

        def cudnn():
            for wi, bi in zip(w, b):
                F.conv2d(x, wi, bi)
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            ms = per_launch_ms(cudnn, args.launches)
            res[f'F.conv2d_tf32_{"on" if tf32 else "off"}'] = dict(
                ms=round(ms, 4), gbs=round(HBM_BYTES / ms / 1e6, 1))
        torch.backends.cudnn.allow_tf32 = False
        # agreement of the two at this shape
        got = head([x])
        ref = [F.conv2d(x.double(), wi.double(), bi.double()) for wi, bi in zip(w, b)]
        res['max_rel_err_vs_fp64'] = max(
            float((g.double() - r).abs().max() / r.abs().max())
            for g, r in zip((got[0][0], got[1][0], got[2][0]), ref))
    out['head'] = res
    out['head_bytes'] = HBM_BYTES

    # share of a whole sample: lifting + neck (+ head), as bench.py runs them
    share = {}
    for name, t, agg, neck_cls in (('waymo_mv', 1, 'mean', modules.OutdoorImVoxelNeck),
                                   ('waymo_10sweep', 2, 'concat', modules.DfMNeck)):
        feats, meta = syn.make_waymo_sample(200, t, 5)
        feats = feats.cuda()
        neck = neck_cls(64, 256, num_frames=2) if neck_cls is modules.DfMNeck \
            else neck_cls(64, 256)
        neck.load_state_dict(syn.make_neck_params(np.random.RandomState(5), neck.state_dict()))
        neck = neck.cuda().eval()

        class Host(modules.MultiViewDfMFeatureTransformation):
            n_voxels, voxel_range = syn.WAYMO_N_VOXELS, syn.WAYMO_RANGE
            temporal_aggregate, valid_sample, neck_3d = agg, True, neck
        host = Host()

        def lift_neck():
            return host.feature_transformation(feats[None], [meta], 5, t)[0]

        def lift_neck_head():
            return head([lift_neck()])
        # the two loops alternate three times; medians.  Their difference is within the run-to-run
        # spread of a 25-60 ms sample, so the head's share is its own kernel time over the sample
        with torch.no_grad():
            per_launch_ms(lift_neck_head, 3, warmup=2)
            a, c = [], []
            for _ in range(3):
                a.append(per_launch_ms(lift_neck, 10, warmup=0))
                c.append(per_launch_ms(lift_neck_head, 10, warmup=0))
        a, c = float(np.median(a)), float(np.median(c))
        share[name] = dict(lift_neck_ms=round(a, 3), lift_neck_head_ms=round(c, 3),
                           head_kernel_share=round(res['head1x1_tc']['ms'] / c, 5))
    out['sample'] = share
    print(json.dumps(out))


if __name__ == '__main__':
    main()
