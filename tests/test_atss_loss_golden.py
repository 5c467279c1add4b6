"""CPU: the torch restatement tests/atss_loss_oracle.py reproduces tests/golden/atss_loss.npz, which
the reference's own LIGAATSSHead and ATSS3DCenterAssigner code wrote
(tests/golden/make_atss_loss_golden.py): the targets bit for bit in fp32, the 15 loss values and
the gradients with respect to the 15 head outputs to the last few ulp."""
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import modules
from depth_from_motion_b200 import synthetic as syn
from tests import atss_loss_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'atss_loss.npz')
WEIGHTS = (0.7, 1.3, 0.9)
KEYS = ('loss_cls', 'loss_bbox', 'loss_centerness')


def _cfg():
    head = modules.LIGAATSSHead(**syn.KITTI_ATSS_HEAD)
    return modules._atss_loss_config(head)


@pytest.mark.parametrize('name', list(syn.ATSS_LOSS_GOLDEN_CASES))
def test_restatement_reproduces_reference_golden(name):
    g = np.load(GOLDEN)
    cfg = _cfg()
    feat_pad, pads, ngt, kw, seed = syn.ATSS_LOSS_GOLDEN_CASES[name]
    feat = syn.atss_feat_sizes(*feat_pad)
    cls, box, ctr, gts, labels = syn.make_atss_loss_case(seed, feat, ngt, pads, **kw)
    tg = O.targets(feat, cfg['strides'], cfg['octave_base_scale'], gts, labels, pads, cfg)
    for k in ('labels', 'label_weights', 'bbox_targets', 'centerness_targets'):
        got = torch.stack([t[k] for t in tg]).numpy()
        np.testing.assert_array_equal(got, g[f'{name}.{k}'], err_msg=k)
    pos = (g[f'{name}.labels'] >= 0) & (g[f'{name}.labels'] < 3)
    np.testing.assert_array_equal(g[f'{name}.bbox_weights'],
                                  np.repeat(pos[..., None], 4, -1).astype(np.float32))
    assert sum(max(t['num_pos'], 1) for t in tg) == int(g[f'{name}.num_total_pos'])
    ins = [[t.clone().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
    ref = O.losses(*ins, tg, feat, cfg['strides'], cfg['octave_base_scale'], cfg)
    for key in KEYS:
        got = np.array([v.item() for v in ref[key]], np.float32)
        np.testing.assert_allclose(got, g[f'{name}.{key}'], rtol=4e-7, atol=1e-12, err_msg=key)
    sum(WEIGHTS[k] * (1 + lv / 10) * ref[key][lv]
        for k, key in enumerate(KEYS) for lv in range(len(feat))).backward()
    for k, ts in zip(('grad_cls', 'grad_bbox', 'grad_centerness'), ins):
        for lv, t in enumerate(ts):
            want = g[f'{name}.{k}.{lv}']
            np.testing.assert_allclose(t.grad.numpy(), want, rtol=4e-7,
                                       atol=1e-6 * float(np.abs(want).max() + 1e-30),
                                       err_msg=f'{k}.{lv}')
