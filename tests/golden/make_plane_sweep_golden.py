"""Generates ``plane_sweep_fp64.npz`` in this directory: the UNMODIFIED reference
``build_dfm_cost`` (mmdet3d/models/backbones/dfm_backbone.py, executed verbatim through
oracle/ref_loader.py) run with float64 as torch's default dtype on fp64 inputs, for the
geometries of ``tests/test_plane_sweep.py::PIN_CASES`` on a 32 x 64 map with 4 channels and 8
planes.  Runs only where the reference tree is available:

    python tests/golden/make_plane_sweep_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from tests import plane_sweep_check as PS  # noqa: E402
from tests.test_plane_sweep import PIN_CASES, small  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ref = load_reference()
    out = {}
    for i, name in enumerate(PIN_CASES):
        cur, prev = syn.white_noise_pair(600 + i, 4, 32, 64)
        g, depths = small(name)
        vol = PS.oracle_volume(cur, prev, depths, g, ref.build_dfm_cost)
        out[f'{name}.cur'] = cur.numpy()
        out[f'{name}.prev'] = prev.numpy()
        out[f'{name}.volume'] = vol.numpy()
    np.savez_compressed(os.path.join(HERE, 'plane_sweep_fp64.npz'), **out)


if __name__ == '__main__':
    main()
