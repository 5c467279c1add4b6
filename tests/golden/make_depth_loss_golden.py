"""Generates ``depth_loss.npz`` in this directory by running the UNMODIFIED reference
``DepthHead`` (dense_heads/depth_head.py, the class executed verbatim through
oracle/ref_loader.py's ``reference_class``) in fp32 on the CPU: its ``upsample_cost``
(``nn.Upsample``, x4 trilinear, align_corners) from a low-res leaf, then its ``loss`` as
``DfM.forward_train`` calls it (detectors/dfm.py:348-357), then autograd.

Per case of ``tests/depth_loss_oracle.GOLDEN_CASES`` the fixture stores the loss, the gradient
with respect to the low-res logits [n, 1, D, H, W] and the gradient with respect to the dense
volume [n, fD, fH, fW] (zeros where the reference's autograd gives none: with no masked pixel
its loss is the Python float 0.).  Inputs regenerate from the seeds.  Runs only where the
reference tree is available, and reproduces the fixture bit for bit:

    python tests/golden/make_depth_loss_golden.py
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.ref_loader import reference_class  # noqa: E402
from tests import depth_loss_oracle as O  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def run_reference(name):
    cfg, cost, depth, fg, preds, samples = O.golden_inputs(name)
    DepthHead = reference_class('mmdet3d/models/dense_heads/depth_head.py', 'DepthHead',
                                dict(torch=torch, nn=nn, F=F, dist=dist))
    g = O.GOLDEN_SHAPE
    head = DepthHead(dict(mode='UD', num_bins=g['D'] * g['f'], min_depth=O.MIN_DEPTH,
                          max_depth=O.MAX_DEPTH), with_convs=False, depth_loss=cfg,
                     downsample_factor=g['f'], num_views=1)
    head.depth_samples = samples
    leaf = cost.clone().requires_grad_()
    vol = head.upsample_cost(leaf).flatten(start_dim=0, end_dim=1)
    vol.retain_grad()
    loss = head.loss(preds, vol, depth, depth_fgmask_img=fg)
    if isinstance(loss, torch.Tensor):
        loss.backward()
    else:
        loss = torch.tensor(loss, dtype=torch.float32)
    zero = torch.zeros_like
    return dict(loss=loss.detach().numpy().astype(np.float32),
                grad_cost=(leaf.grad if leaf.grad is not None else zero(leaf)).numpy(),
                grad_volume=(vol.grad if vol.grad is not None else zero(vol)).numpy())


def main():
    torch.set_num_threads(1)
    out = {}
    for name in O.GOLDEN_CASES:
        for k, v in run_reference(name).items():
            out[f'{name}.{k}'] = v
    np.savez_compressed(os.path.join(HERE, 'depth_loss.npz'), **out)
    print('wrote', len(out), 'arrays')


if __name__ == '__main__':
    main()
