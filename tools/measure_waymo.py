#!/usr/bin/env python
"""Times the Waymo-side rows (SURVEY.md 8a: a6 lifting, a7 necks) at the shipped sizes
(configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync[_10sweeps].py):
T*Nv x [64, 208, 312] features -> [64(*T), 220, 300, 12] voxels -> BEV [256, 300, 220].
Prints one JSON line; run on an H100."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from depth_from_motion_b200 import modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402


def timeit(fn, n=3):
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
    rng = np.random.RandomState(0)
    out = {}
    n_voxels, vrange = [220, 300, 12], [-35.0, -75.0, -2.0, 75.0, 75.0, 4.0]
    for t in (1, 2):
        nv = 5
        feats = torch.from_numpy(rng.standard_normal((t * nv, 64, 208, 312)).astype(np.float32)).cuda()
        mats = []
        for f in range(t):
            for v in range(nv):
                yaw = (v - 2) * 0.7
                r = np.array([[np.cos(yaw), np.sin(yaw), 0], [-np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
                l2c = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64) @ r
                ext = np.eye(4)
                ext[:3, :3] = l2c
                ext[:3, 3] = l2c @ np.array([-1.0 * f, 0.0, -1.5])
                k = np.array([[1335., 0, 624, 0], [0, 1335., 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
                mats.append(k @ ext)
        meta = dict(ori_lidar2img=np.array(mats), input_shape=(832, 1248),
                    img_shape=[(832, 1248, 3)] * (t * nv), scale_factor=1.0, flip=False)
        agg = 'concat' if t == 2 else 'mean'
        ms = timeit(lambda: modules.multiview_lift(feats, meta, n_voxels, vrange, nv, t, agg))
        out_bytes = 64 * t * 220 * 300 * 12 * 4
        in_bytes = feats.numel() * 4
        out[f'lift_T{t}'] = dict(ms=round(ms, 3), gbs=round((in_bytes + out_bytes) / ms / 1e6, 1))
    for name, mod, cin in (('OutdoorImVoxelNeck', modules.OutdoorImVoxelNeck(64, 256), 64),
                           ('DfMNeck', modules.DfMNeck(64, 256, num_frames=2), 128)):
        mod.load_state_dict(syn.make_neck_params(rng, mod.state_dict()))
        mod = mod.cuda().eval()
        x = torch.from_numpy(rng.standard_normal((1, cin, 220, 300, 12)).astype(np.float32)).cuda()
        ms = timeit(lambda: mod(x), n=1)
        flops = 3.212e12 if cin == 64 else 7.649e12
        out[name] = dict(ms=round(ms, 1), tflops=round(flops / ms / 1e9, 2), impl='wgmma K-outer conv (conv_tc_neck.cuh)')
    print(json.dumps(out))


if __name__ == '__main__':
    main()
