"""CPU: the torch restatement tests/anchor_loss_oracle.py reproduces tests/golden/anchor_loss.npz,
which the reference's own loss code wrote (tests/golden/make_anchor_loss_golden.py), bit for bit
in fp32: targets, loss values and the gradients with respect to the three head outputs."""
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import modules
from depth_from_motion_b200 import synthetic as syn
from tests import anchor_loss_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'anchor_loss.npz')
WEIGHTS = (0.7, 1.3, 0.9, 1.1)


def _config(kind, with_iou):
    if kind == 'liga':
        head = modules.LIGAAnchor3DHead(
            num_classes=3, in_channels=64, feat_channels=64,
            norm_cfg=dict(type='GN', num_groups=32), anchor_generator=syn.KITTI_ANCHOR_GENERATOR,
            dir_offset=syn.KITTI_DIR_OFFSET, assign_per_class=True, diff_rad_by_sin=True,
            train_cfg=syn.KITTI_TRAIN_CFG,
            **dict(syn.KITTI_LOSSES, loss_iou=syn.KITTI_LOSSES['loss_iou'] if with_iou else None))
    else:
        head = modules.Anchor3DHead(
            num_classes=3, in_channels=256, anchor_generator=syn.WAYMO_ANCHOR_GENERATOR,
            dir_offset=syn.WAYMO_DIR_OFFSET, train_cfg=syn.WAYMO_TRAIN_CFG, **syn.WAYMO_LOSSES)
    return head, modules._loss_config(head, kind == 'liga')


@pytest.mark.parametrize('name', list(syn.ANCHOR_LOSS_GOLDEN_CASES))
def test_restatement_reproduces_reference_golden(name):
    g = np.load(GOLDEN)
    kind, ny, nx, ngt, kw, with_iou, seed = syn.ANCHOR_LOSS_GOLDEN_CASES[name]
    head, cfg = _config(kind, with_iou)
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, 'cpu')
    cls, box, dirc, gts, labels = syn.make_anchor_loss_case(
        seed, anchors.numpy(), ny, nx, cfg['num_sizes'], cfg['num_rots'], cfg['num_classes'],
        ngt, **kw)
    tg = O.targets(anchors, cfg['num_sizes'], cfg['num_rots'], gts, labels, cfg)
    for k in ('labels', 'label_weights', 'bbox_targets', 'dir_targets'):
        got = torch.stack([t[k] for t in tg]).numpy()
        np.testing.assert_array_equal(got, g[f'{name}.{k}'], err_msg=k)
    pos = (g[f'{name}.labels'] >= 0) & (g[f'{name}.labels'] < 3)
    np.testing.assert_array_equal(g[f'{name}.dir_weights'], pos.astype(np.float32))
    np.testing.assert_array_equal(g[f'{name}.bbox_weights'],
                                  np.repeat(pos[..., None], 7, -1).astype(np.float32))
    assert sum(max(t['num_pos'], 1) for t in tg) == int(g[f'{name}.num_total_pos'])
    ins = [t.clone().requires_grad_() for t in (cls, box, dirc)]
    ref = O.losses(*ins, tg, anchors, cfg)
    keys = ['loss_cls', 'loss_bbox', 'loss_dir'] + (['loss_iou'] if cfg['with_iou'] else [])
    assert sorted(ref) == sorted(keys)
    for k in keys:
        assert ref[k].item() == g[f'{name}.{k}'].item(), k
    sum(w * ref[k] for w, k in zip(WEIGHTS, keys)).backward()
    for k, t in zip(('grad_cls', 'grad_bbox', 'grad_dir'), ins):
        np.testing.assert_array_equal(t.grad.numpy(), g[f'{name}.{k}'], err_msg=k)
