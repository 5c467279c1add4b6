"""Records the ``model`` dicts of every shipped DfM / MultiViewDfM config, as
``registry.Config.fromfile`` parses them, into detector_configs.json, so that the detector
construction tests run without the reference tree.  Runs where the reference is available
(DFM_REFERENCE_ROOT):

    python tests/golden/make_detector_configs.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import registry  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = ['dfm_r34_1x8_kitti-3d-3class.py',
           'dfm_r34_1x8_kitti-3d-3class_wophotodist.py',
           'dfm_r34_1x8_kitti-3d-3class_wophotodist_wodistnorm.py',
           'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py',
           'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py']


def main():
    out = {}
    for name in CONFIGS:
        cfg = registry.Config.fromfile(os.path.join(REFERENCE_ROOT, 'configs/dfm', name))
        out[name] = json.loads(json.dumps(dict(cfg.model), default=list))
    with open(os.path.join(HERE, 'detector_configs.json'), 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == '__main__':
    main()
