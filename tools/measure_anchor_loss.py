"""Times ``loss`` + ``backward`` of both anchor heads on CUDA against the torch restatement
(tests/anchor_loss_oracle.py, fp32) composed on the same GPU, with the native per-stage split
(assignment, loss pass) from the library's profiling record.  Prints one JSON line with the card
name and power limit.

    KITTI: B = 1, the shipped LIGAAnchor3DHead config, 20 GT
    Waymo: B = 2, the shipped Anchor3DHead config, 250 GT per sample

    python tools/measure_anchor_loss.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import capi  # noqa: E402
from tests import anchor_loss_oracle as O  # noqa: E402
from tests import test_anchor_loss as T  # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f'unknown ({e})'


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def measure(name, iters):
    head, liga, cfg, anchors, outs, gts, labels, metas = T._run_case(name)

    def native():
        for o in outs:
            o.grad = None
        got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, labels, metas)
        sum(v[0] for v in got.values()).backward()

    def restated():
        ins = [o.detach().requires_grad_() for o in outs]
        tg = O.targets(anchors, cfg['num_sizes'], cfg['num_rots'], gts, labels, cfg)
        sum(O.losses(*ins, tg, anchors, cfg).values()).backward()

    t_native = _time(native, iters)
    t_ref = _time(restated, max(2, iters // 5))
    capi.profile_enable(True)
    capi.profile_report()
    native()
    torch.cuda.synchronize()
    stages = {k.split('@')[0]: round(v['ms'], 4) for k, v in capi.profile_report().items()}
    capi.profile_enable(False)
    return dict(ms_native=round(t_native, 3), ms_restatement=round(t_ref, 3),
                speedup=round(t_ref / t_native, 2), stages_ms=stages)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('measure_anchor_loss: no CUDA device')
    out = dict(tool='measure_anchor_loss', card=_card(),
               kitti_b1_20gt=measure('kitti_b1', args.iters),
               waymo_b2_250gt=measure('waymo_b2', args.iters))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
