#!/usr/bin/env python
"""Times the stride-2 hourglass convs (conv1 32->64, conv3 64->64) of both towers at the
benchmarked KITTI shape (D = 112, 384 x 1248 features) on the two routes of conv1, alternately in
one process: the cluster-shared bricks (default for the stereo tower) and the input-channel
slices (DFM_S2_KSLICE=1, fed by TMA from a pre-split copy of the input).  The mono tower's conv1
and conv3 run as input-channel slices on both and are a control for run-to-run drift.  Per layer
it prints ms per step (CUDA events around every launch, presplit and slice-reduce passes
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
    # presplit rows carry the input depth, conv rows the output depth
    if cls.startswith('presplit<32>'):
        return 'conv1', 'stereo' if dz == D else 'mono'
    if cls.startswith(('conv_tc_ks<32->64,s2', 'conv_tc_cl<32->64,s2')):
        return 'conv1', 'stereo' if dz == D // 2 else 'mono'
    if cls.startswith(('conv_tc_ks<64->64,s2', 'conv_tc_cl<64->64,s2')):
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
    models = {}
    for route in ('kslice', 'cluster'):
        if route == 'kslice':
            os.environ['DFM_S2_KSLICE'] = '1'
        else:
            os.environ.pop('DFM_S2_KSLICE', None)
        m = modules.DfMBackbone(in_channels=C, depth_cfg=cfg).cuda().eval()
        m.load_state_dict(params, strict=True)
        with torch.no_grad():
            m(cur, prev, copy.deepcopy(metas))     # weights are built (route fixed) on first use
        models[route] = m
    os.environ.pop('DFM_S2_KSLICE', None)
    torch.cuda.synchronize()
    ms = {r: {} for r in models}
    rows = {r: {} for r in models}
    with torch.no_grad():
        for _ in range(ROUNDS):
            for route, m in models.items():
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
                    ms[route].setdefault(lt, []).append(v['ms'] / STEPS)
                    rows[route].setdefault(lt, set()).add(k)
    out = dict(card=card(), shape=dict(D=D, feature_hw=[H, W]), rounds=ROUNDS,
               steps_per_round=STEPS, layers={})
    for route in models:
        for (layer, tower), per_round in sorted(ms[route].items()):
            # rows of one layer are summed per round (conv + presplit / slice reduce)
            n = len(rows[route][(layer, tower)])
            sums = [sum(per_round[i:i + n]) for i in range(0, len(per_round), n)]
            t = sorted(sums)[len(sums) // 2]
            nbytes = algorithmic_bytes(layer, tower)
            out['layers'][f'{layer}.{tower}.{route}'] = dict(
                ms=round(t, 4), ms_rounds=[round(s, 4) for s in sums],
                rows=sorted(rows[route][(layer, tower)]),
                algorithmic_gb=round(nbytes / 1e9, 3), gbs=round(nbytes / t / 1e6, 1),
                share_of_hbm=round(nbytes / t / 1e6 / (HBM_TBS * 1e3), 3))
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
