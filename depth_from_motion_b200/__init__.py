"""depth_from_motion_b200 -- H100-native (sm_90a) DfM plane-sweep cost-volume path.

Host-side mirror of the reference's plugin interface (registry + module
classes) over the C-ABI CUDA library ``libdfm_b200.so`` (``include/dfm_b200.h``).
"""
from . import capi, checkpoint  # noqa: F401
from .modules import (CostLogits, DepthHead, DfM, DfMBackbone,  # noqa: F401
                      DfMNeck, FrustumToVoxel, MultiViewDfM, OutdoorImVoxelNeck, build_dfm_cost, conv3d,
                      multiview_lift)
from .registry import (BACKBONES, DETECTORS, HEADS, NECKS, Config,  # noqa: F401
                       build_backbone, build_detector, build_head, build_neck,
                       register_into_mmdet)

__version__ = '0.1.0'
