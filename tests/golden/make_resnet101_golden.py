"""Generates ``resnet101_dcn.npz`` in this directory from an implementation independent of the
tests' restatement: ``torchvision.models.resnet101(weights=None)`` (no download) with the conv2
of every layer3 / layer4 Bottleneck replaced by a module that runs
``torchvision.ops.deform_conv2d(x, offset, weight, stride=s, padding=1, mask=sigmoid(m))`` on the
output of its ``conv_offset`` (3x3, 27 channels, bias) -- mmcv's ``ModulatedDeformConv2dPack``
(DCNv2, deform_groups 1), which both MultiViewDfM (Waymo) configs put in layer3 / layer4 with
``fallback_on_stride=False``.  torchvision's Bottleneck puts the stride in conv2, as mmdet's
style 'pytorch' does, and its parameter names are mmdet's, so the synthetic state_dict loads
with ``strict=True`` (``fc`` removed).

    python tests/golden/make_resnet101_golden.py

Inputs regenerate from the seed (``synthetic.make_resnet101_case``); the fixture stores their
checksums, a random sample of every output level, the first / last rows and columns of the odd
case's outputs, and the state_dict's keys and shapes.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

# must match tests/test_resnet101.py
CASES = {'small': (81, 2, 64, 96), 'odd': (82, 1, 70, 134)}
EDGE_CASES = ('odd',)
N_SAMPLE = 4096


class DeformConv2dPack(nn.Module):
    """mmcv ModulatedDeformConv2dPack (3x3, no bias, deform_groups 1) on torchvision's op."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        from torchvision.ops import deform_conv2d
        self.op = deform_conv2d
        self.weight = nn.Parameter(torch.zeros(cout, cin, 3, 3))
        self.conv_offset = nn.Conv2d(cin, 27, 3, stride, 1, bias=True)
        self.stride = stride

    def forward(self, x):
        o = self.conv_offset(x)
        return self.op(x, o[:, :18], self.weight, None, stride=self.stride, padding=1,
                       mask=torch.sigmoid(o[:, 18:]))


def build():
    import torchvision
    m = torchvision.models.resnet101(weights=None)
    del m.fc
    for name in ('layer3', 'layer4'):
        for blk in getattr(m, name):
            c = blk.conv2
            blk.conv2 = DeformConv2dPack(c.in_channels, c.out_channels, c.stride[0])
    return m.eval()


def forward(m, img):
    x = m.maxpool(m.relu(m.bn1(m.conv1(img))))
    outs = []
    for name in ('layer1', 'layer2', 'layer3', 'layer4'):
        x = getattr(m, name)(x)
        outs.append(x)
    return outs


def main():
    from depth_from_motion_b200 import synthetic as syn
    torch.set_grad_enabled(False)
    arrs = {}
    for name, (seed, b, h, w) in CASES.items():
        img, sd = syn.make_resnet101_case(seed, h, w, b)
        m = build()
        m.load_state_dict(sd, strict=True)
        if name == 'small':
            arrs['state_keys'] = np.array(list(m.state_dict()))
            arrs['state_shapes'] = np.array([','.join(str(n) for n in v.shape)
                                             for v in m.state_dict().values()])
        arrs[f'{name}_img_sums'] = np.array([img.double().sum().item(),
                                             img.double().abs().sum().item()])
        arrs[f'{name}_w_abs'] = np.array(sum(v.double().abs().sum().item() for v in sd.values()))
        outs = forward(m, img)
        for lvl, o in enumerate(outs):
            n = o[0].numel()
            idx = torch.from_numpy(np.random.RandomState(seed + 100 * (lvl + 1)).randint(0, n, N_SAMPLE))
            arrs[f'{name}_out{lvl}_sample'] = torch.stack(
                [o[i].reshape(-1)[idx] for i in range(b)]).numpy()
            if name in EDGE_CASES:
                th, tw = o.shape[2:]
                arrs[f'{name}_out{lvl}_rows'] = o[:, :, [0, th - 1], :].numpy()
                arrs[f'{name}_out{lvl}_cols'] = o[:, :, :, [0, tw - 1]].numpy()
            print(name, lvl, tuple(o.shape), float(o.abs().max()), float(o.abs().mean()))
    np.savez_compressed(os.path.join(HERE, 'resnet101_dcn.npz'), **arrs)


if __name__ == '__main__':
    main()
