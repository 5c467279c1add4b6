"""Times ``LIGAATSSHead.loss`` + ``backward`` (dfm_atss_loss_*) against the torch restatement
(tests/atss_loss_oracle.py, fp32, targets and losses under autograd) on the same GPU, at the
shipped config and the 320 x 1280 training shape with 20 GT per image, B = 1 and 2.  Prints the
card's name and power limit, one JSON line per batch size, and, from a torch.profiler trace of
one native call, its kernel launches and any host synchronisation.  With ``--out DIR`` the
trace is also written there as Chrome JSON.

    python tools/measure_atss_loss.py [--iters 50] [--out DIR]
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
from tests import atss_loss_oracle as O  # noqa: E402

TRAIN = (320, 1280)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 \
        else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--out', default=None, help='also write the profiler traces here')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('measure_atss_loss: no CUDA device')
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    feat = syn.atss_feat_sizes(*TRAIN)
    head = modules.LIGAATSSHead(**syn.KITTI_ATSS_HEAD)
    cfg = modules._atss_loss_config(head)
    print('card:', card())
    for B in (1, 2):
        pads = [TRAIN] * B
        cls, box, ctr, gts, labels = syn.make_atss_loss_case(61 + B, feat, [20] * B, pads)
        outs = [[t.cuda().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
        gts = [g.cuda() for g in gts]
        labels = [lab.cuda() for lab in labels]
        metas = [dict(pad_shape=(h, w, 3)) for h, w in pads]

        def native():
            got = head.loss(*outs, gts, labels, metas)
            sum(sum(v) for v in got.values()).backward()

        def restatement():
            tg = O.targets(feat, cfg['strides'], cfg['octave_base_scale'], gts, labels, pads, cfg)
            got = O.losses(*outs, tg, feat, cfg['strides'], cfg['octave_base_scale'], cfg)
            sum(sum(v) for v in got.values()).backward()

        t_nat, t_ref = timed(native, a.iters), timed(restatement, max(a.iters // 5, 3))
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            got = head.loss(*outs, gts, labels, metas)
            torch.cuda.synchronize()
        if a.out:
            prof.export_chrome_trace(os.path.join(a.out, f'atss_loss_b{B}.pt.trace.json'))
        ev = prof.events()
        kernels = sorted({e.name for e in ev if e.device_type.name == 'CUDA' and
                          'at_' in e.name and 'kernel' in e.name})
        n_launch = sum(1 for e in ev if e.device_type.name == 'CUDA' and e.name in kernels)
        syncs = [e.name for e in ev if 'Synchronize' in e.name and
                 e.name != 'cudaDeviceSynchronize']
        print(json.dumps(dict(batch=B, gt_per_image=20, shape=list(TRAIN),
                              native_loss_backward_ms=round(t_nat, 3),
                              restatement_loss_backward_ms=round(t_ref, 3),
                              native_kernels=kernels, native_kernel_launches=n_launch,
                              stream_syncs_in_call=syncs, card=card())))


if __name__ == '__main__':
    main()
