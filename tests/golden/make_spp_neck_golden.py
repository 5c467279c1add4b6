"""Generates ``spp_neck.npz`` in this directory by running the UNMODIFIED reference
``SPPUNetNeck`` (mmdet3d/models/necks/spp_unet_neck.py, built in place by oracle/ref_loader.py
with the shipped KITTI ``neck`` block, configs/dfm/dfm_r34_1x8_kitti-3d-3class.py; its
SyncBatchNorm runs in eval on the CPU).  Runs only where the reference tree is available:

    python tests/golden/make_spp_neck_golden.py

Inputs regenerate from the seed (``synthetic.make_spp_neck_case``); the fixture stores their
checksums.  Cases (image H x W):
  * 256 x 512: the smallest legal shape, the 64-pool of f4 leaves 1 x 2 cells;
  * 300 x 536: H/4 = 75 is odd (ragged conv tiles, floor-dropped pool rows).
Per case: the four branch maps before upsampling in full, and ``stereo_feature`` and
``sem_feature`` each at a seeded sample of indices; for the 300 x 536 case, whose conv tiles are
ragged, also their first / last rows and columns.  (The full maps of both cases would be about
1.5 MB compressed.)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
# must match tests/test_spp_neck.py
CASES = {'small': (41, 256, 512), 'odd': (42, 300, 536)}
EDGE_CASES = ('odd',)
N_SAMPLE = {'stereo': 4096, 'sem': 8192}
NECK_CFG = dict(in_channels=[3, 64, 128, 128, 128], start_level=2, sem_channels=[128, 32],
                stereo_channels=[32, 32], with_upconv=True, cat_img_feature=True,
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))


def sample_index(seed, what, h, w):
    """Flat indices into [32, h, w] of the stored sample of `what` ('stereo' / 'sem')."""
    off = 1000 if what == 'stereo' else 2000
    return np.random.RandomState(seed + off).randint(0, 32 * h * w, N_SAMPLE[what])


def main():
    ns = load_reference()
    arrs = {}
    for name, (seed, h, w) in CASES.items():
        feats, sd = syn.make_spp_neck_case(seed, h, w)
        m = ns.SPPUNetNeck(**NECK_CFG).eval()
        m.load_state_dict(sd, strict=True)
        if name == 'small':
            arrs['state_keys'] = np.array(list(m.state_dict()))
            arrs['state_shapes'] = np.array([','.join(str(n) for n in v.shape)
                                             for v in m.state_dict().values()])
        with torch.no_grad():
            stereo, sem = m(feats)
            for i, br in enumerate(m.spp_branches):
                arrs[f'{name}_spp{i}'] = br(feats[-1])[0].numpy()
        for what, t in (('stereo', stereo[0].numpy()), ('sem', sem[0].numpy())):
            th, tw = t.shape[1:]
            arrs[f'{name}_{what}_sample'] = t.reshape(-1)[sample_index(seed, what, th, tw)]
            if name in EDGE_CASES:
                arrs[f'{name}_{what}_rows'] = t[:, [0, th - 1], :]
                arrs[f'{name}_{what}_cols'] = t[:, :, [0, tw - 1]]
        arrs[f'{name}_feat_sums'] = np.array([[f.double().sum().item(), f.double().abs().sum().item()]
                                              for f in feats])
        arrs[f'{name}_w_abs'] = np.float64(sum(v.double().abs().sum().item() for v in sd.values()))
        print(name, tuple(stereo.shape), tuple(sem.shape), float(stereo.abs().max()),
              float(sem.abs().max()))
    np.savez_compressed(os.path.join(HERE, 'spp_neck.npz'), **arrs)


if __name__ == '__main__':
    main()
