"""Times ``DfMImitation.loss`` + ``backward`` (dfm_imitation_loss_*) against the torch
restatement (tests/imitation_loss_oracle.py in fp32 under autograd: the mask, the dense conv over
the positive rows and the loss) on the same GPU, at the shipped KITTI shape ([B, 64, 304, 288]
BEV and [B, 32, 5, 304, 288] volume features) with B = 1 and 2 and 0 / 20 / 60 GT per sample.
Prints the card's name and power limit and one JSON line per case with both times, both peak
memory increments over the inputs and the native call's kernel launches from a torch.profiler
trace.

    python tools/measure_imitation_loss.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from tests import imitation_loss_oracle as O  # noqa: E402

KEYS = ('spatial_features_2d', 'volume_features')
CFGS = [dict(lidar_feature_layer=k, stereo_feature_layer=k, normalize='cw_scale',
             layer='conv2d' if k == KEYS[0] else 'conv3d', channel=64 if k == KEYS[0] else 32,
             kernel_size=1, use_relu=False, mode='inbox', loss_weight=1.0) for k in KEYS]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 \
        else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t) / iters * 1e3
    return ms, (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('measure_imitation_loss: no CUDA device')
    print('card:', card())
    m = modules.DfMImitation(CFGS, syn.KITTI_ANCHOR_GENERATOR, 10).cuda().train()
    convs = list(m.conv_imitation)
    ax, ay = O.anchor_centres(syn.KITTI_ANCHOR_GENERATOR, 304, 288, 'cuda')
    for B in (1, 2):
        for G in (0, 20, 60):
            case = syn.make_imitation_case(90 + B * 7 + G, B, G)
            xs = {k: case['stereo'][k].cuda().requires_grad_() for k in KEYS}
            ts = {k: case['teacher'][k].cuda() for k in KEYS}
            gt = [g.cuda() for g in case['gt']]
            scales = [m.norm_imitation[k].scale for k in KEYS]

            def native():
                sum(m.loss(xs, ts, gt)).backward()

            def restatement():
                inbox = O.inbox_mask(ax, ay, gt)
                losses, _, _ = O.imitation_loss(
                    [xs[k] for k in KEYS], [ts[k] for k in KEYS], [c.weight for c in convs],
                    [c.bias for c in convs], scales, inbox, [1.0, 1.0], 10.0, False)
                sum(losses).backward()

            t_nat, mem_nat = timed(native, a.iters)
            t_ref, mem_ref = timed(restatement, max(a.iters // 5, 3))
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                native()
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if e.device_type.name == 'CUDA' and
                  'dfm::im_' in e.name]
            pos = m.debug_tensor('counts').tolist()
            print(json.dumps(dict(batch=B, gt_per_sample=G, positives=pos,
                                  native_loss_backward_ms=round(t_nat, 3),
                                  restatement_loss_backward_ms=round(t_ref, 3),
                                  native_peak_mib=round(mem_nat, 1),
                                  restatement_peak_mib=round(mem_ref, 1),
                                  native_kernel_launches=len(ev),
                                  workspace_mib=round(m.workspace() / 2**20, 2), card=card())))


if __name__ == '__main__':
    main()
