#!/usr/bin/env python
"""Times FrustumToVoxel (SURVEY.md section 8(f) row 1) at the shipped KITTI size
(configs/dfm/dfm_r34_1x8_kitti-3d-3class.py: stereo_feat [32,112,96,312], softmax
[448,384,1248], voxels 20x304x288) with the materialised softmax volume (the reference's
argument) and with the fused logits path, plus the per-kernel split.  Prints one JSON line;
run on an H100."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402


def timeit(fn, n=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    d = int(os.environ.get('DFM_PLANES', '112'))
    c = syn.make_frustum_case(51, 384, 1248, d, (288, 304, 20))
    m = modules.FrustumToVoxel()
    m.load_state_dict(c['params'], strict=True)
    m = m.cuda().eval()
    m.coordinates_3d, m.depth_cfg = c['coordinates_3d'], c['depth_cfg']
    stereo, cost, sem = c['stereo'].cuda(), c['cost'].cuda(), c['sem'].cuda()
    head = modules.DepthHead(depth_cfg=dict(mode='UD', num_bins=4 * d, min_depth=2,
                                            max_depth=59.6), with_convs=False)
    from oracle import dfm_oracle as O  # depth table only
    head.depth_samples = O.depth_samples(c['depth_cfg'])
    _, sm, _ = head(cost)
    out = {'planes': d}
    out['materialised_ms'] = round(timeit(lambda: m(stereo, sm, c['metas'], sem)), 3)
    out['depth_head_with_volumes_ms'] = round(timeit(lambda: head(cost)), 3)
    out['depth_head_preds_only_ms'] = round(
        timeit(lambda: head(cost, return_volumes=False)), 3)
    del sm
    logits = modules.CostLogits(cost)
    out['fused_ms'] = round(timeit(lambda: m(stereo, logits, c['metas'], sem)), 3)
    lp = modules.CostLogits(cost, depth_samples=head.depth_samples)
    out['fused_with_depth_preds_ms'] = round(timeit(lambda: m(stereo, lp, c['metas'], sem)), 3)
    capi.profile_enable(True)
    m(stereo, logits, c['metas'], sem)
    torch.cuda.synchronize()
    out['kernels'] = {k: round(v['ms'], 3) for k, v in capi.profile_report().items()}
    capi.profile_enable(False)
    nvox = 20 * 304 * 288
    out['conv_tflops'] = round(2 * 27 * 64 * 32 * nvox / 1e9 /
                               max(v for k, v in out['kernels'].items() if 'conv' in k), 1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
