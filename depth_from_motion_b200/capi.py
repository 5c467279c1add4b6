"""ctypes binding of ``include/dfm_b200.h`` (the C-ABI shared library).

The library is built in-tree by ``__graft_entry__.build()`` /
``depth_from_motion_b200/build.py`` as ``depth_from_motion_b200/libdfm_b200.so``.
There is no fallback: if the library is missing, or no sm_90 GPU is visible
when a compute entry point is called, the caller gets a ``RuntimeError``.
"""
import ctypes
import os
from ctypes import (POINTER, c_char_p, c_double, c_float, c_int, c_longlong,
                    c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('DFM_B200_LIB') or os.path.join(_HERE, 'libdfm_b200.so')

DFM_OK = 0
DFM_CONV_AUTO, DFM_CONV_SIMT, DFM_CONV_TC, DFM_CONV_TC_NECK, DFM_CONV_TC_NECK_DHW = 0, 1, 2, 3, 4
DFM_OUT_COST, DFM_OUT_STEREO, DFM_OUT_MONO = 1, 2, 4
DFM_LAYOUT_NCDHW, DFM_LAYOUT_DHWC = 0, 1

# every symbol include/dfm_b200.h declares (tests/test_host_logic.py checks the
# header against this list and against the built library)
SYMBOLS = (
    'dfm_last_error', 'dfm_version', 'dfm_device_info', 'dfm_launch_counters',
    'dfm_sync_check', 'dfm_profile_enable', 'dfm_profile_report',
    'dfm_backbone_create', 'dfm_backbone_destroy', 'dfm_backbone_set_param',
    'dfm_backbone_set_depths', 'dfm_backbone_missing_params',
    'dfm_backbone_workspace_bytes', 'dfm_backbone_forward',
    'dfm_backbone_forward_host', 'dfm_backbone_prefetch_host',
    'dfm_backbone_cost_device',
    'dfm_backbone_stereo_feat_device',
    'dfm_backbone_debug_tensor', 'dfm_op_build_cost_volume', 'dfm_op_conv3d',
    'dfm_depth_head_forward', 'dfm_multiview_lift', 'dfm_multiview_lift_cl', 'dfm_neck_create',
    'dfm_neck_destroy', 'dfm_neck_set_param', 'dfm_neck_missing_params',
    'dfm_neck_forward', 'dfm_neck_forward_cl', 'dfm_frustum_create', 'dfm_frustum_destroy',
    'dfm_frustum_set_param', 'dfm_frustum_missing_params', 'dfm_frustum_forward',
    'dfm_pipeline_forward_host', 'dfm_pipeline_submit_host', 'dfm_pipeline_wait',
    'dfm_pipeline_prefetch_host',
    'dfm_bev_hourglass_create', 'dfm_bev_hourglass_destroy', 'dfm_bev_hourglass_set_param',
    'dfm_bev_hourglass_missing_params', 'dfm_bev_hourglass_forward',
    'dfm_anchor_head_create', 'dfm_anchor_head_destroy', 'dfm_anchor_head_set_param',
    'dfm_anchor_head_missing_params', 'dfm_anchor_head_forward', 'dfm_voxel_sample',
    'dfm_backbone_forward_cl', 'dfm_stereo_tail_create', 'dfm_stereo_tail_destroy',
    'dfm_stereo_tail_set_param', 'dfm_stereo_tail_missing_params', 'dfm_stereo_tail_forward',
    'dfm_neck_debug_tensor', 'dfm_frustum_debug_tensor', 'dfm_bev_hourglass_debug_tensor',
    'dfm_anchor_head_debug_tensor',
    'dfm_anchor3d_head_create', 'dfm_anchor3d_head_destroy', 'dfm_anchor3d_head_set_param',
    'dfm_anchor3d_head_missing_params', 'dfm_anchor3d_head_forward',
    'dfm_spp_neck_create', 'dfm_spp_neck_destroy', 'dfm_spp_neck_set_param',
    'dfm_spp_neck_missing_params', 'dfm_spp_neck_forward', 'dfm_spp_neck_debug_tensor',
    'dfm_fpn_create', 'dfm_fpn_destroy', 'dfm_fpn_set_param', 'dfm_fpn_missing_params',
    'dfm_fpn_forward', 'dfm_fpn_debug_tensor',
    'dfm_liga_resnet_create', 'dfm_liga_resnet_destroy', 'dfm_liga_resnet_set_param',
    'dfm_liga_resnet_missing_params', 'dfm_liga_resnet_forward', 'dfm_liga_resnet_debug_tensor',
    'dfm_resnet101_create', 'dfm_resnet101_destroy', 'dfm_resnet101_set_param',
    'dfm_resnet101_missing_params', 'dfm_resnet101_forward', 'dfm_resnet101_debug_tensor',
    'dfm_box_post_create', 'dfm_box_post_destroy', 'dfm_box_post_forward',
    'dfm_box_post_debug_tensor', 'dfm_op_rotated_iou', 'dfm_image_prep',
    'dfm_multiview_lift_views', 'dfm_multiview_lift_views_cl', 'dfm_view_fingerprint',
    'dfm_views_equal', 'dfm_fpn_set_num_images', 'dfm_liga_resnet_set_num_images',
    'dfm_resnet101_set_num_images', 'dfm_kitti_eval_create', 'dfm_kitti_eval_destroy',
    'dfm_kitti_eval_forward', 'dfm_kitti_eval_debug_tensor', 'dfm_op_eval_rotated_iou',
    'dfm_op_let_iou', 'dfm_kitti_eval_set_overlap_limit', 'dfm_kitti_eval_workspace',
    'dfm_waymo_kitti_convert', 'dfm_anchor_loss_create', 'dfm_anchor_loss_destroy',
    'dfm_anchor_loss_forward', 'dfm_anchor_loss_finish', 'dfm_anchor_loss_debug_tensor',
    'dfm_depth_loss_create', 'dfm_depth_loss_destroy', 'dfm_depth_loss_workspace',
    'dfm_depth_loss_forward', 'dfm_depth_loss_debug_tensor',
    'dfm_atss_loss_create', 'dfm_atss_loss_destroy', 'dfm_atss_loss_forward',
    'dfm_atss_loss_finish', 'dfm_atss_loss_debug_tensor',
    'dfm_imitation_loss_create', 'dfm_imitation_loss_destroy', 'dfm_imitation_loss_workspace',
    'dfm_imitation_loss_forward', 'dfm_imitation_loss_finish', 'dfm_imitation_loss_backward',
    'dfm_imitation_loss_debug_tensor',
)

DFM_IMAGE_PREP_CROP, DFM_IMAGE_PREP_RESCALE = 0, 1


class Geometry(ctypes.Structure):
    """``dfm_geometry_t``."""
    _fields_ = [('cam2img', c_double * 16), ('cur2prev', c_double * 16),
                ('crop_x', c_double), ('crop_y', c_double),
                ('scale', c_double), ('org_w', c_double), ('flip', c_int),
                ('reserved', c_int)]


class BackboneDesc(ctypes.Structure):
    """``dfm_backbone_desc_t``."""
    _fields_ = [('in_channels', c_int), ('cv_channels', c_int),
                ('feat_h', c_int), ('feat_w', c_int), ('num_planes', c_int),
                ('cost_sample_factor', c_int), ('feat_sample_factor', c_int),
                ('conv_impl', c_int)]


class LiftDesc(ctypes.Structure):
    """``dfm_lift_desc_t``."""
    _fields_ = [('num_frames', c_int), ('num_views', c_int),
                ('channels', c_int), ('feat_h', c_int), ('feat_w', c_int),
                ('n_voxels', c_int * 3), ('scale_x', c_float),
                ('scale_y', c_float), ('crop_x', c_float), ('crop_y', c_float),
                ('flip', c_int), ('input_h', c_int), ('input_w', c_int),
                ('concat', c_int)]


class NeckDesc(ctypes.Structure):
    """``dfm_neck_desc_t``."""
    _fields_ = [('in_channels', c_int), ('out_channels', c_int),
                ('num_frames', c_int), ('nx', c_int), ('ny', c_int),
                ('nz', c_int), ('conv_impl', c_int)]


class FrustumDesc(ctypes.Structure):
    """``dfm_frustum_desc_t``."""
    _fields_ = [(n, c_int) for n in
                ('num_3dconvs', 'cv_channels', 'out_channels', 'in_sem_channels',
                 'sem_atten_feat', 'stereo_atten_feat', 'cat_img_feature',
                 'num_planes', 'feat_h', 'feat_w', 'sem_h', 'sem_w',
                 'depth_factor', 'nx', 'ny', 'nz')] + \
               [('depth_min', c_float), ('depth_max', c_float),
                ('conv_impl', c_int)]


class BevDesc(ctypes.Structure):
    """``dfm_bev_desc_t``."""
    _fields_ = [(n, c_int) for n in ('in_channels', 'out_channels', 'ny', 'nx', 'conv_impl')]


class AnchorHeadDesc(ctypes.Structure):
    """``dfm_anchor_head_desc_t``."""
    _fields_ = [(n, c_int) for n in
                ('in_channels', 'feat_channels', 'num_convs', 'cls_channels', 'reg_channels',
                 'dir_channels', 'ny', 'nx', 'conv_impl')]


class Anchor3DHeadDesc(ctypes.Structure):
    """``dfm_anchor3d_head_desc_t``."""
    _fields_ = [(n, c_int) for n in
                ('feat_channels', 'cls_channels', 'reg_channels', 'dir_channels', 'ny', 'nx',
                 'conv_impl')]


class FpnDesc(ctypes.Structure):
    """``dfm_fpn_desc_t``."""
    _fields_ = [('in_channels', c_int * 4), ('out_channels', c_int), ('level_h', c_int * 4),
                ('level_w', c_int * 4), ('num_images', c_int), ('conv_impl', c_int)]


class LigaResNetDesc(ctypes.Structure):
    """``dfm_liga_resnet_desc_t``."""
    _fields_ = [(n, c_int) for n in ('height', 'width', 'num_images', 'conv_impl')]


class ResNet101Desc(ctypes.Structure):
    """``dfm_resnet101_desc_t``."""
    _fields_ = [(n, c_int) for n in ('height', 'width', 'num_images', 'conv_impl')]


class BoxPostDesc(ctypes.Structure):
    """``dfm_box_post_desc_t``."""
    _fields_ = [(n, c_int) for n in ('num_classes', 'num_anchors', 'ny', 'nx', 'batch',
                                     'use_sigmoid', 'nms_pre', 'max_num')] + \
               [(n, c_float) for n in ('score_thr', 'nms_thr', 'dir_offset', 'dir_limit_offset')]


class AnchorLossDesc(ctypes.Structure):
    """``dfm_anchor_loss_desc_t``."""
    _fields_ = [(n, c_int) for n in ('num_classes', 'num_sizes', 'num_rotations', 'ny', 'nx',
                                     'batch', 'assign_per_class', 'diff_rad_by_sin',
                                     'use_direction_classifier', 'with_iou', 'liga')] + \
               [(n, c_float * 8) for n in ('pos_iou_thr', 'neg_iou_thr', 'min_pos_iou')] + \
               [(n, c_float) for n in ('pos_weight', 'gamma', 'alpha', 'beta')] + \
               [('loss_weight', c_float * 4)] + \
               [(n, c_float) for n in ('dir_offset', 'dir_limit_offset',
                                       'normalizer_clamp_value')]


class DepthLossDesc(ctypes.Structure):
    """``dfm_depth_loss_desc_t``."""
    _fields_ = [(n, c_int) for n in ('num_images', 'num_planes', 'height', 'width', 'factor',
                                     'dense')] + \
               [(n, c_float) for n in ('min_depth', 'max_depth', 'alpha', 'gamma', 'fg_weight',
                                       'bg_weight')] + \
               [('balanced', c_int), ('loss_weight', c_float)]


class AtssLossDesc(ctypes.Structure):
    """``dfm_atss_loss_desc_t``."""
    _fields_ = [('num_classes', c_int), ('num_levels', c_int), ('strides', c_int * 8),
                ('feat_h', c_int * 8), ('feat_w', c_int * 8), ('batch', c_int), ('topk', c_int),
                ('octave_base_scale', c_float), ('target_stds', c_float * 4),
                ('wh_ratio_clip', c_float), ('giou_eps', c_float), ('gamma', c_float),
                ('alpha', c_float), ('loss_weight', c_float * 3)]


class ImitationLossDesc(ctypes.Structure):
    """``dfm_imitation_loss_desc_t``."""
    _fields_ = [(n, c_int) for n in ('batch', 'ny', 'nx', 'num_pairs')] + \
               [('channels', c_int * 2), ('depth', c_int * 2), ('loss_weight', c_float * 2),
                ('normalizer_clamp_value', c_float)]


class ImagePrepDesc(ctypes.Structure):
    """``dfm_image_prep_desc_t``."""
    _fields_ = [(n, c_int) for n in ('mode', 'num_views', 'src_h', 'src_w', 'crop_x', 'crop_y',
                                     'out_h', 'out_w', 'pad_divisor', 'to_rgb')] + \
               [('mean', c_double * 3), ('std', c_double * 3)]


class KittiEvalDesc(ctypes.Structure):
    """``dfm_kitti_eval_desc_t``."""
    _fields_ = [('num_classes', c_int), ('classes', c_int * 3), ('num_metrics', c_int),
                ('metrics', c_int * 3), ('compute_aos', c_int), ('f32_flags', c_int),
                ('min_overlap', c_double * 18)]


class VoxelSampleDesc(ctypes.Structure):
    """``dfm_voxel_sample_desc_t``."""
    _fields_ = [('channels', c_int), ('nx', c_int), ('ny', c_int), ('nz', c_int),
                ('voxel_range', c_float * 6), ('voxel_size', c_float * 3),
                ('num_depths', c_int), ('out_h', c_int), ('out_w', c_int),
                ('downsample_factor', c_int), ('scale_x', c_float), ('scale_y', c_float),
                ('crop_x', c_float), ('crop_y', c_float), ('flip', c_int), ('img_w', c_int),
                ('aligned', c_int)]


_lib = None


def library_built():
    return os.path.isfile(LIB_PATH)


def lib():
    """Loads the shared library once; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not library_built():
        raise RuntimeError(
            f'{LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; '
            'g.build()"` (nvcc, sm_90a). There is no CPU/PyTorch fallback.')
    L = ctypes.CDLL(LIB_PATH)
    fp, vp, ip = POINTER(c_float), c_void_p, POINTER(c_int)
    L.dfm_last_error.restype = c_char_p
    L.dfm_version.restype = c_int
    L.dfm_device_info.argtypes = [ip, ip, ip, POINTER(c_longlong)]
    L.dfm_launch_counters.argtypes = [POINTER(c_longlong), POINTER(c_longlong)]
    L.dfm_sync_check.argtypes = [vp]
    L.dfm_profile_enable.argtypes = [c_int]
    L.dfm_profile_report.argtypes = [c_char_p, c_int]
    L.dfm_backbone_create.argtypes = [POINTER(BackboneDesc), POINTER(vp)]
    L.dfm_backbone_set_depths.argtypes = [vp, vp, c_int]
    L.dfm_backbone_workspace_bytes.argtypes = [vp]
    L.dfm_backbone_workspace_bytes.restype = c_longlong
    L.dfm_backbone_forward.argtypes = [vp, vp, vp, POINTER(Geometry), vp, vp,
                                       vp, vp]
    L.dfm_backbone_forward_host.argtypes = [vp, vp, vp, POINTER(Geometry),
                                            c_int, vp, vp, vp, vp]
    L.dfm_backbone_prefetch_host.argtypes = [vp, vp, vp]
    L.dfm_pipeline_prefetch_host.argtypes = [vp, vp, vp, vp, ctypes.c_longlong]
    L.dfm_backbone_cost_device.argtypes = [vp]
    L.dfm_backbone_cost_device.restype = vp
    L.dfm_backbone_stereo_feat_device.argtypes = [vp]
    L.dfm_backbone_stereo_feat_device.restype = vp
    L.dfm_op_build_cost_volume.argtypes = [vp, vp, c_int, c_int, c_int, vp,
                                           c_int, c_int, c_int,
                                           POINTER(Geometry), vp, vp]
    L.dfm_op_conv3d.argtypes = [vp, c_int, c_int, c_int, c_int, vp, c_int,
                                POINTER(c_int), POINTER(c_int), c_int, c_int,
                                vp, vp]
    L.dfm_depth_head_forward.argtypes = [vp, vp, c_int, c_int, c_int, c_int,
                                         vp, vp, vp, vp]
    L.dfm_multiview_lift.argtypes = [POINTER(LiftDesc), vp, vp, vp, vp, vp, vp,
                                     vp, vp]
    L.dfm_multiview_lift_cl.argtypes = [POINTER(LiftDesc), vp, vp, vp, vp, vp, vp,
                                     vp, vp]
    L.dfm_multiview_lift_views.argtypes = [POINTER(LiftDesc), POINTER(vp), vp, vp, vp, vp, vp,
                                           vp, vp]
    L.dfm_multiview_lift_views_cl.argtypes = [POINTER(LiftDesc), POINTER(vp), vp, vp, vp, vp,
                                              vp, vp, vp]
    L.dfm_view_fingerprint.argtypes = [vp, c_int, c_longlong, vp, vp]
    L.dfm_views_equal.argtypes = [POINTER(vp), POINTER(vp), c_int, c_longlong, vp, vp]
    L.dfm_neck_create.argtypes = [POINTER(NeckDesc), POINTER(vp)]
    L.dfm_neck_forward.argtypes = [vp, vp, vp, vp]
    L.dfm_neck_forward_cl.argtypes = [vp, vp, vp, vp]
    L.dfm_frustum_create.argtypes = [POINTER(FrustumDesc), vp, vp, vp,
                                     POINTER(vp)]
    L.dfm_frustum_forward.argtypes = [vp, vp, c_int, vp, vp, vp, vp, vp,
                                      POINTER(c_double), c_int, c_int, vp, vp]
    L.dfm_pipeline_forward_host.argtypes = [vp, vp, vp, vp, vp, POINTER(Geometry),
                                            POINTER(c_double), c_int, c_int, vp, vp, vp,
                                            vp, vp]
    L.dfm_pipeline_submit_host.argtypes = [vp, vp, vp, vp, vp, POINTER(Geometry),
                                           POINTER(c_double), c_int, c_int, vp, vp, vp, vp]
    L.dfm_pipeline_wait.argtypes = [vp]
    L.dfm_bev_hourglass_create.argtypes = [POINTER(BevDesc), POINTER(vp)]
    L.dfm_bev_hourglass_forward.argtypes = [vp, vp, vp, vp, vp]
    L.dfm_anchor_head_create.argtypes = [POINTER(AnchorHeadDesc), POINTER(vp)]
    L.dfm_anchor_head_forward.argtypes = [vp, vp, vp, vp, vp, vp]
    L.dfm_anchor3d_head_create.argtypes = [POINTER(Anchor3DHeadDesc), POINTER(vp)]
    L.dfm_anchor3d_head_forward.argtypes = [vp, vp, vp, vp, vp, vp]
    L.dfm_backbone_forward_cl.argtypes = [vp, vp, vp, POINTER(Geometry), vp, vp, vp, vp]
    L.dfm_stereo_tail_create.argtypes = [c_int, c_int, c_int, POINTER(vp)]
    L.dfm_stereo_tail_forward.argtypes = [vp, vp, vp, vp, vp]
    L.dfm_spp_neck_create.argtypes = [c_int, c_int, c_int, POINTER(vp)]
    L.dfm_spp_neck_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dfm_fpn_create.argtypes = [POINTER(FpnDesc), POINTER(vp)]
    L.dfm_fpn_forward.argtypes = [vp, POINTER(vp), POINTER(vp), vp]
    L.dfm_liga_resnet_create.argtypes = [POINTER(LigaResNetDesc), POINTER(vp)]
    L.dfm_liga_resnet_forward.argtypes = [vp, vp, POINTER(vp), vp]
    L.dfm_resnet101_create.argtypes = [POINTER(ResNet101Desc), POINTER(vp)]
    L.dfm_resnet101_forward.argtypes = [vp, vp, POINTER(vp), vp]
    for f in ('fpn', 'liga_resnet', 'resnet101'):
        getattr(L, f'dfm_{f}_set_num_images').argtypes = [vp, c_int]
    # the parameterised handle families share destroy / set_param / missing_params
    for f in ('backbone', 'neck', 'frustum', 'bev_hourglass', 'anchor_head', 'anchor3d_head',
              'stereo_tail', 'spp_neck', 'fpn', 'liga_resnet', 'resnet101'):
        getattr(L, f'dfm_{f}_destroy').argtypes = [vp]
        getattr(L, f'dfm_{f}_set_param').argtypes = [vp, c_char_p, vp, c_longlong]
        getattr(L, f'dfm_{f}_missing_params').argtypes = [vp]
    for f in ('backbone', 'neck', 'frustum', 'bev_hourglass', 'anchor_head', 'spp_neck', 'fpn',
              'liga_resnet', 'resnet101', 'box_post'):
        getattr(L, f'dfm_{f}_debug_tensor').argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_box_post_create.argtypes = [POINTER(BoxPostDesc), vp, POINTER(vp)]
    L.dfm_box_post_destroy.argtypes = [vp]
    L.dfm_box_post_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dfm_op_rotated_iou.argtypes = [vp, vp, c_int, vp, vp]
    L.dfm_anchor_loss_create.argtypes = [POINTER(AnchorLossDesc), vp, POINTER(vp)]
    L.dfm_anchor_loss_destroy.argtypes = [vp]
    L.dfm_anchor_loss_forward.argtypes = [vp] * 14
    L.dfm_anchor_loss_finish.argtypes = [vp] * 5
    L.dfm_anchor_loss_debug_tensor.argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_depth_loss_create.argtypes = [POINTER(DepthLossDesc), POINTER(vp)]
    L.dfm_depth_loss_destroy.argtypes = [vp]
    L.dfm_depth_loss_workspace.argtypes = [vp, POINTER(c_longlong)]
    L.dfm_depth_loss_forward.argtypes = [vp] * 10
    L.dfm_depth_loss_debug_tensor.argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_atss_loss_create.argtypes = [POINTER(AtssLossDesc), POINTER(vp)]
    L.dfm_atss_loss_destroy.argtypes = [vp]
    L.dfm_atss_loss_forward.argtypes = [vp] * 14
    L.dfm_atss_loss_finish.argtypes = [vp] * 5
    L.dfm_atss_loss_debug_tensor.argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_imitation_loss_create.argtypes = [POINTER(ImitationLossDesc), POINTER(vp)]
    L.dfm_imitation_loss_destroy.argtypes = [vp]
    L.dfm_imitation_loss_workspace.argtypes = [vp, POINTER(c_longlong)]
    L.dfm_imitation_loss_forward.argtypes = [vp] * 10 + [c_int, vp, vp]
    L.dfm_imitation_loss_finish.argtypes = [vp, vp, c_int, vp, vp, vp]
    L.dfm_imitation_loss_backward.argtypes = [vp] * 7
    L.dfm_imitation_loss_debug_tensor.argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_voxel_sample.argtypes = [POINTER(VoxelSampleDesc), vp, vp, POINTER(c_double), vp, vp]
    L.dfm_kitti_eval_create.argtypes = [POINTER(KittiEvalDesc), POINTER(vp)]
    L.dfm_kitti_eval_destroy.argtypes = [vp]
    L.dfm_kitti_eval_forward.argtypes = [vp, c_int, c_int, c_int, c_longlong] + [vp] * 10 + [vp]
    L.dfm_kitti_eval_debug_tensor.argtypes = [vp, c_char_p, vp, c_longlong, vp]
    L.dfm_op_eval_rotated_iou.argtypes = [vp, vp, c_int, c_int, c_int, vp, vp]
    L.dfm_op_let_iou.argtypes = [vp, vp, c_int, c_int, vp, vp]
    L.dfm_kitti_eval_set_overlap_limit.argtypes = [vp, c_longlong]
    L.dfm_kitti_eval_workspace.argtypes = [vp, POINTER(c_longlong), POINTER(c_longlong),
                                           POINTER(c_int)]
    L.dfm_waymo_kitti_convert.argtypes = [c_int, c_int] + [vp] * 5 + [POINTER(c_float)] + \
        [vp] * 4
    L.dfm_image_prep.argtypes = [POINTER(ImagePrepDesc), vp, vp, vp]
    _lib = L
    return L


def check(rc, what):
    """Turns a DFM_ERR_* return code into a RuntimeError with the C message."""
    if rc != DFM_OK:
        msg = lib().dfm_last_error().decode('utf-8', 'replace')
        raise RuntimeError(f'{what} failed (code {rc}): {msg}')


def sync_check(stream=None):
    """Synchronise and raise on any asynchronous kernel failure."""
    check(lib().dfm_sync_check(c_void_p(stream or 0)), 'dfm_sync_check')


def profile_enable(on=True):
    check(lib().dfm_profile_enable(int(on)), 'dfm_profile_enable')


def profile_report():
    """dict: kernel class -> {launches, ms, flops} since the last report."""
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib().dfm_profile_report(buf, len(buf)), 'dfm_profile_report')
    return json.loads(buf.value.decode() or '{}')


def launch_counters():
    a, b = c_longlong(0), c_longlong(0)
    lib().dfm_launch_counters(ctypes.byref(a), ctypes.byref(b))
    return a.value, b.value
