"""Generates ``liga_resnet.npz`` in this directory by running the UNMODIFIED reference
``LIGAResNet`` and ``LigaBasicBlock`` (mmdet3d/models/backbones/liga_resnet.py, executed verbatim
through oracle/ref_loader.py's ``reference_class`` on the stand-ins below for mmcv's conv / norm
builders and mmdet's ``ResNet`` base) with the shipped KITTI ``backbone`` block
(configs/dfm/dfm_r34_1x8_kitti-3d-3class.py; its SyncBN runs in eval on the CPU).  Runs only
where the reference tree is available:

    python tests/golden/make_liga_resnet_golden.py

Inputs regenerate from the seed (``synthetic.make_liga_resnet_case``); the fixture stores their
checksums.  Cases (image B x H x W):
  * 2 x 64 x 160: two images in one call;
  * 1 x 70 x 134: odd sizes (ceil(H / 2) = 35, then 18 x 34; ragged tiles everywhere).
Per case and output: a seeded sample of indices per image; for the odd case also the first / last
rows and columns of every output.
"""
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from depth_from_motion_b200 import synthetic as syn  # noqa: E402
from oracle.ref_loader import _BaseModule, reference_class  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
# must match tests/test_liga_resnet.py
CASES = {'small': (51, 2, 64, 160), 'odd': (52, 1, 70, 134)}
EDGE_CASES = ('odd',)
N_SAMPLE = 4096
BACKBONE_CFG = dict(depth=34, num_stages=4, strides=(1, 2, 1, 1), dilations=(1, 1, 2, 4),
                    out_indices=(0, 1, 2, 3), style='pytorch', frozen_stages=-1,
                    norm_cfg=dict(type='SyncBN', requires_grad=True), norm_eval=False,
                    with_max_pool=False, block_with_final_relu=False,
                    num_channels_factor=(1, 2, 2, 2))


class _ResLayer(nn.Sequential):
    """Restatement of mmdet 2.x ``mmdet/models/utils/res_layer.py::ResLayer`` (not in the
    reference tree), the builder of ``ResNet.make_res_layer``: a 1x1 conv + norm ``downsample``
    when the stride or the width changes (``avg_down`` adds an AvgPool2d in front and moves the
    stride there), the first block with ``stride``, the rest with stride 1; every other keyword
    goes to every block."""

    def __init__(self, block, inplanes, planes, num_blocks, stride=1, avg_down=False,
                 conv_cfg=None, norm_cfg=dict(type='BN'), downsample_first=True, **kwargs):
        assert downsample_first
        downsample = None
        if stride != 1 or inplanes != planes * block.expansion:
            downsample = []
            conv_stride = stride
            if avg_down:
                conv_stride = 1
                downsample.append(nn.AvgPool2d(kernel_size=stride, stride=stride,
                                               ceil_mode=True, count_include_pad=False))
            downsample.extend([
                _build_conv_layer(conv_cfg, inplanes, planes * block.expansion, kernel_size=1,
                                  stride=conv_stride, bias=False),
                _build_norm_layer(norm_cfg, planes * block.expansion)[1]])
            downsample = nn.Sequential(*downsample)
        layers = [block(inplanes=inplanes, planes=planes, stride=stride, downsample=downsample,
                        conv_cfg=conv_cfg, norm_cfg=norm_cfg, **kwargs)]
        inplanes = planes * block.expansion
        for _ in range(1, num_blocks):
            layers.append(block(inplanes=inplanes, planes=planes, stride=1, conv_cfg=conv_cfg,
                                norm_cfg=norm_cfg, **kwargs))
        super().__init__(*layers)


def _build_conv_layer(cfg, *args, **kwargs):
    """Stand-in for mmcv.cnn.build_conv_layer: None / Conv2d -> nn.Conv2d."""
    assert cfg is None or cfg.get('type') == 'Conv2d', cfg
    return nn.Conv2d(*args, **kwargs)


def _build_norm_layer(cfg, num_features, postfix=''):
    """Stand-in for mmcv.cnn.build_norm_layer with BN / SyncBN (abbreviation 'bn'; SyncBN in
    eval on one device is BatchNorm2d)."""
    assert cfg['type'] in ('BN', 'SyncBN'), cfg
    layer = nn.BatchNorm2d(num_features)
    for p in layer.parameters():
        p.requires_grad = cfg.get('requires_grad', True)
    return 'bn' + str(postfix), layer


class _ResNetBase(_BaseModule):
    """Stand-in for the parts of mmdet 2.x ``ResNet`` that ``LIGAResNet`` inherits:
    ``make_res_layer`` (a ``ResLayer``), the ``norm1`` property and ``_freeze_stages``
    (``frozen_stages = -1``: nothing is frozen)."""

    def make_res_layer(self, **kwargs):
        return _ResLayer(**kwargs)

    def make_stage_plugins(self, plugins, stage_idx):
        raise NotImplementedError('plugins')

    @property
    def norm1(self):
        return getattr(self, self.norm1_name)

    def _freeze_stages(self):
        assert self.frozen_stages == -1


def load_liga_resnet():
    """The reference ``LIGAResNet`` and ``LigaBasicBlock`` (backbones/liga_resnet.py), executed
    verbatim on the stand-ins above."""
    import torch.utils.checkpoint as cp
    rel = 'mmdet3d/models/backbones/liga_resnet.py'
    ns = dict(nn=nn, cp=cp, build_conv_layer=_build_conv_layer,
              build_norm_layer=_build_norm_layer, build_plugin_layer=None,
              BaseModule=_BaseModule, ResNet=_ResNetBase)
    ns['LigaBasicBlock'] = reference_class(rel, 'LigaBasicBlock', ns)
    ns['LigaBottleneck'] = reference_class(rel, 'LigaBottleneck', ns)
    return types.SimpleNamespace(LIGAResNet=reference_class(rel, 'LIGAResNet', ns),
                                 LigaBasicBlock=ns['LigaBasicBlock'])


def sample_index(seed, level, n):
    """Flat indices into one image's output `level` ([C, h, w], n elements)."""
    return np.random.RandomState(seed + 100 * (level + 1)).randint(0, n, N_SAMPLE)


def main():
    ns = load_liga_resnet()
    arrs = {}
    for name, (seed, b, h, w) in CASES.items():
        img, sd = syn.make_liga_resnet_case(seed, h, w, b)
        m = ns.LIGAResNet(**BACKBONE_CFG).eval()
        m.load_state_dict(sd, strict=True)
        if name == 'small':
            arrs['state_keys'] = np.array(list(m.state_dict()))
            arrs['state_shapes'] = np.array([','.join(str(n) for n in v.shape)
                                             for v in m.state_dict().values()])
        with torch.no_grad():
            outs = m(img)
        for lvl, o in enumerate(outs):
            o = o.numpy()
            arrs[f'{name}_out{lvl}_sample'] = np.stack(
                [o[i].reshape(-1)[sample_index(seed, lvl, o[i].size)] for i in range(b)])
            if name in EDGE_CASES:
                th, tw = o.shape[2:]
                arrs[f'{name}_out{lvl}_rows'] = o[:, :, [0, th - 1], :]
                arrs[f'{name}_out{lvl}_cols'] = o[:, :, :, [0, tw - 1]]
        arrs[f'{name}_img_sums'] = np.array([img.double().sum().item(),
                                             img.double().abs().sum().item()])
        arrs[f'{name}_w_abs'] = np.float64(sum(v.double().abs().sum().item() for v in sd.values()))
        print(name, [tuple(o.shape) for o in outs], [float(o.abs().max()) for o in outs])
    np.savez_compressed(os.path.join(HERE, 'liga_resnet.npz'), **arrs)


if __name__ == '__main__':
    main()
