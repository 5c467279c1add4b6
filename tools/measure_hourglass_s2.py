#!/usr/bin/env python
"""Times the stride-2 hourglass convs of both towers at the benchmarked KITTI shape (D = 112,
384 x 1248 features): conv1 (32->64) on cluster-shared bricks and conv3 (64->64) on input-channel
slices.  Per layer it prints ms per step (CUDA events around every launch, the slice-reduce pass
included), GB/s of the algorithmic bytes (inputs read once, output written once) and their share
of the 3.35 TB/s data-sheet HBM bandwidth, next to the card name and power limit.  Run on an
H100."""
import copy
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from depth_from_motion_b200 import capi, modules  # noqa: E402
from depth_from_motion_b200 import synthetic as syn  # noqa: E402

H, W, D, C = 384, 1248, 112, 32
HBM_TBS = 3.35
ROUNDS, STEPS = 4, 10


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit not readable'


def layer_of(key):
    """('conv1' | 'conv3', tower) of a profile row, or None."""
    cls, _, shape = key.partition('@')
    dz = int(shape.split('x')[0]) if shape else 0
    if cls.startswith('conv_tc_cl<32->64,s2'):
        return 'conv1', 'stereo' if dz == D // 2 else 'mono'
    if cls.startswith('conv_tc_ks<64->64,s2'):
        return 'conv3', 'stereo' if dz == D // 4 else 'mono'
    return None


def algorithmic_bytes(layer, tower):
    ho, wo = H // 4, W // 4
    planes = D if tower == 'stereo' else 40      # the mono tower computes 16 + 8 + 16 planes
    if layer == 'conv1':
        # reads gn1(raw1) (every computed plane) + relu(gn0(raw0)) (stereo: every plane, mono:
        # the 3-plane z-class tensor), writes b1
        t0 = planes if tower == 'stereo' else 3
        return (planes + t0) * ho * wo * 32 * 4 + planes // 8 * ho * wo * 64 * 4
    # conv3 reads relu(gn2(b2)) at half resolution and writes b3 at quarter resolution
    return planes // 8 * ho * wo * 64 * 4 + planes // 64 * ho * wo * 64 * 4


def main():
    cur, prev, metas, params = syn.make_kitti_pair(100, H, W, D)
    metas[0]['cam2img'] = syn.KITTI_P2.astype('float32').tolist()
    cur, prev = cur.cuda(), prev.cuda()
    cfg = syn.depth_cfg_for(D)
    m = modules.DfMBackbone(in_channels=C, depth_cfg=cfg).cuda().eval()
    m.load_state_dict(params, strict=True)
    ms, rows = {}, {}
    with torch.no_grad():
        for _ in range(ROUNDS):
            m(cur, prev, copy.deepcopy(metas))
            torch.cuda.synchronize()
            capi.profile_enable(True)
            capi.profile_report()
            for _ in range(STEPS):
                m(cur, prev, metas)
            torch.cuda.synchronize()
            rep = capi.profile_report()
            capi.profile_enable(False)
            for k, v in rep.items():
                lt = layer_of(k)
                if lt is None:
                    continue
                ms.setdefault(lt, []).append(v['ms'] / STEPS)
                rows.setdefault(lt, set()).add(k)
    out = dict(card=card(), shape=dict(D=D, feature_hw=[H, W]), rounds=ROUNDS,
               steps_per_round=STEPS, layers={})
    for (layer, tower), per_round in sorted(ms.items()):
        t = sorted(per_round)[len(per_round) // 2]
        nbytes = algorithmic_bytes(layer, tower)
        out['layers'][f'{layer}.{tower}'] = dict(
            ms=round(t, 4), ms_rounds=[round(s, 4) for s in per_round],
            rows=sorted(rows[(layer, tower)]),
            algorithmic_gb=round(nbytes / 1e9, 3), gbs=round(nbytes / t / 1e6, 1),
            share_of_hbm=round(nbytes / t / 1e6 / (HBM_TBS * 1e3), 3))
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
