# A flat python config in the style of configs/dfm/*.py, for registry.Config.fromfile.
import math  # noqa: F401  (modules are not config entries)

num_planes = 72
depth_range = (2.0, 59.6)
model = dict(
    type='DfM',
    backbone_stereo=dict(type='DfMBackbone', in_channels=32, cv_channels=32, num_hg=1,
                         cost_sample_factor=4,
                         norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)),
    depth_cfg=dict(mode='UD', num_bins=num_planes * 4, depth_min=depth_range[0],
                   depth_max=depth_range[1], downsample_factor=4),
    neck_3d=dict(type='DfMNeck', in_channels=64, out_channels=256, num_frames=2))
voxel_size = [0.2 * s for s in (1, 1, 2)]


def _helper():  # callables are not config entries
    return None
