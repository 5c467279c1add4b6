"""Times get_bboxes of the anchor heads on the GPU: the C entry point (dfm_box_post_forward,
CUDA events over repeated calls), the module call (head.get_bboxes, including its one
device-to-host read of the counts) and the torch restatement tests/box_post_oracle.py on the
same GPU tensors (one sample), at the KITTI (304 x 288) and Waymo (300 x 220) grids with B = 1
and B = 2.
Prints the card name and power limit first.

    python tools/measure_box_post.py [--iters 50]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from tests import box_post_oracle as BP  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                               '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'measuring needs a GPU'
    print('card:', card())
    for name, ny, nx, gen, cfg, off in (
            ('kitti', 304, 288, syn.KITTI_ANCHOR_GENERATOR, syn.KITTI_TEST_CFG, syn.KITTI_DIR_OFFSET),
            ('waymo', 300, 220, syn.WAYMO_ANCHOR_GENERATOR, syn.WAYMO_TEST_CFG, syn.WAYMO_DIR_OFFSET)):
        for B in (1, 2):
            cases = [syn.make_box_post_case(40 + b, ny, nx) for b in range(B)]
            cls, box, dirc = (torch.stack([c[i] for c in cases]).cuda() for i in range(3))
            head = modules.Anchor3DHead(num_classes=3, in_channels=256, anchor_generator=gen,
                                        dir_offset=off, test_cfg=cfg)
            metas = [{}] * B
            out = head.get_bboxes([cls], [box], [dirc], metas)       # creates the handle
            capi.sync_check()
            L, bp = capi.lib(), head._box_post
            mx = cfg['max_num']
            ob = torch.empty((B, mx, 7), device='cuda')
            osc = torch.empty((B, mx), device='cuda')
            ol = torch.empty((B, mx), device='cuda', dtype=torch.int32)
            oc = torch.empty((B,), device='cuda', dtype=torch.int32)
            p, s = modules._ptr, modules._stream()

            def c_call():
                capi.check(L.dfm_box_post_forward(bp._handle, p(cls), p(box), p(dirc), p(ob),
                                                  p(osc), p(ol), p(oc), s), 'forward')
            for _ in range(5):
                c_call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                c_call()
            e1.record()
            torch.cuda.synchronize()
            c_ms = e0.elapsed_time(e1) / args.iters
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                head.get_bboxes([cls], [box], [dirc], metas)
            torch.cuda.synchronize()
            m_ms = (time.perf_counter() - t0) * 1e3 / args.iters
            o_txt = ''
            if B == 1:   # the restatement's greedy NMS is a host loop: one sample, one call
                anchors = modules.grid_anchors(gen, ny, nx, 'cuda')
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with torch.no_grad():
                    BP.get_bboxes_single(cls[0], box[0], dirc[0], anchors, cfg, 3, True, off)
                torch.cuda.synchronize()
                o_txt = f', torch restatement {(time.perf_counter() - t0) * 1e3:.0f} ms'
            n = [len(o[0]) for o in out]
            print(f'{name} {ny}x{nx} B={B}: C entry {c_ms:.3f} ms ({c_ms / B:.3f} ms/sample), '
                  f'module {m_ms:.3f} ms{o_txt}; boxes {n}', flush=True)
            capi.profile_enable(True)
            capi.profile_report()
            for _ in range(args.iters):
                c_call()
            torch.cuda.synchronize()
            rep = capi.profile_report()
            capi.profile_enable(False)
            print('  per-stage ms/call:', {k.split('@')[0]: round(v['ms'] / v['launches'], 4)
                                           for k, v in rep.items()}, flush=True)


if __name__ == '__main__':
    main()
