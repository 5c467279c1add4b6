"""Times ``DepthHead.loss`` + ``backward`` on CUDA (``CostLogits`` form, the shipped
balanced_focal config) against the reference's computation restated in torch on the same GPU:
``F.interpolate`` (x4 trilinear, align_corners) of the low-res logits, then the loss of
tests/depth_loss_oracle.py's dense form, under autograd.  Shipped KITTI training shape: cost
logits [1, 1, 72, 80, 320], volume [288, 320, 1280].  Reports ms per call, the native per-stage
split from the library's profiling record, and each arm's peak ``max_memory_allocated`` above
its inputs.  Prints one JSON line with the card name and power limit.

    sparse:    synthetic scan-line depth map, about 5 % of the pixels carry a depth
    all_valid: every pixel carries a depth (those inside [2, 59.6] are masked)

    python tools/measure_depth_loss.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import capi, modules  # noqa: E402
from tests import depth_loss_oracle as O  # noqa: E402
from tests import test_depth_loss as T  # noqa: E402


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


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)


def measure(density, iters):
    head = T._head(O.SHIPPED_LOSS, T.SHIPPED['D'])
    cost, depth, fg, preds = T._shipped_case(1, density)
    samples = head.depth_samples.cuda()
    x = cost.clone().requires_grad_()

    def native():
        x.grad = None
        head.loss(preds, modules.CostLogits(x), depth, fg).backward()

    def restated():
        x.grad = None
        O.dense_loss(T._upsample(x), depth, fg, samples, O.SHIPPED_LOSS, preds).backward()

    t_native = _time(native, iters)
    t_ref = _time(restated, max(2, iters // 2))
    mem_native, mem_ref = _peak(native), _peak(restated)
    capi.profile_enable(True)
    capi.profile_report()
    native()
    torch.cuda.synchronize()
    stages = {k.split('@')[0]: round(v['ms'], 4) for k, v in capi.profile_report().items()}
    capi.profile_enable(False)
    masked = ((depth > O.MIN_DEPTH) & (depth < O.MAX_DEPTH)).float().mean().item()
    return dict(masked_fraction=round(masked, 4), ms_native=round(t_native, 3),
                ms_restatement=round(t_ref, 3), speedup=round(t_ref / t_native, 2),
                peak_mib_native=mem_native, peak_mib_restatement=mem_ref,
                workspace_mib=round(head._depth_loss.workspace() / 2**20, 1), stages_ms=stages)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('measure_depth_loss: no CUDA device')
    out = dict(tool='measure_depth_loss', card=_card(),
               sparse=measure(0.05, args.iters), all_valid=measure(1.0, args.iters))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
