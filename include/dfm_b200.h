/*
 * dfm_b200.h -- C ABI of the H100-native (sm_90a) DfM plane-sweep cost-volume path.
 *
 * The reference (Tai-Wang/Depth-from-Motion @ e2321189) has no FFI: its hot path
 * is a chain of PyTorch calls inside mmcv-registry modules.  This header is the
 * boundary a maintainer binds instead of those chains; every entry point names the
 * reference interface it replaces (file:line relative to the reference checkout).
 * INTEGRATION.md shows the ctypes binding used by depth_from_motion_b200/modules.py
 * and the ten-line patch that makes the reference's own modules call it.
 *
 * Conventions
 *   - plain C types only; all tensors are dense fp32, layouts stated per argument;
 *   - pointers named d_* are CUDA device pointers, h_* are host pointers;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     device entry points are asynchronous on that stream, *_host entry points
 *     synchronise the stream before returning;
 *   - every function returns DFM_OK (0) or a DFM_ERR_* code; dfm_last_error()
 *     returns a thread-local human-readable message for the last failure;
 *   - there is no CPU fallback anywhere behind this ABI.
 */
#ifndef DFM_B200_H_
#define DFM_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define DFM_OK 0
#define DFM_ERR_INVALID 1 /* bad argument / unsupported shape           */
#define DFM_ERR_CUDA 2    /* CUDA runtime error (message has the cause)  */
#define DFM_ERR_STATE 3   /* missing parameter, depths not set, ...      */
#define DFM_ERR_NOGPU 4   /* no sm_90 device visible                     */

/* conv implementation selector (dfm_backbone_desc_t.conv_impl, dfm_op_conv3d) */
#define DFM_CONV_AUTO 0 /* tensor-core (wgmma) kernels where implemented, SIMT else */
#define DFM_CONV_SIMT 1 /* fp32 CUDA-core kernels everywhere (bring-up / cross-check) */
#define DFM_CONV_TC 2   /* wgmma only; error if a layer has no tensor-core kernel     */
#define DFM_CONV_TC_NECK 3 /* dfm_op_conv3d only: force the K-outer wgmma kernel of the BEV
                              necks (64..256 channels, W <= 16, strides (1,1,1) / (1,1,2))  */
#define DFM_CONV_TC_NECK_DHW 4 /* dfm_op_conv3d only: force the same kernel in [D][H][W]
                                  orientation, D cut into windows (stride 1, pad 1, Cin >= 64) */

/* output-selection flags for the *_host entry points */
#define DFM_OUT_COST 1   /* gated depth logits           [1,1,D,Ho,Wo] */
#define DFM_OUT_STEREO 2 /* stereo tower feature         [1,32,D,Ho,Wo] */
#define DFM_OUT_MONO 4   /* mono tower feature           [1,32,D,Ho,Wo] */

const char* dfm_last_error(void);
int dfm_version(void);
/* Reports the visible device; DFM_ERR_NOGPU when there is none. */
int dfm_device_info(int* sm_count, int* cc_major, int* cc_minor, long long* l2_bytes);

/* ------------------------------------------------------------------------------------
 * Geometry of one (cur, prev) pair -- the img_meta fields DfMBackbone.forward reads
 * (mmdet3d/models/backbones/dfm_backbone.py:150-172).
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_geometry {
  double cam2img[16];  /* img_metas[0]['ori_cam2img'], 4x4 row-major              */
  double cur2prev[16]; /* img_metas[0]['cur2prevs'][0], 4x4 row-major            */
  double crop_x;       /* img_metas[0]['crop_offset'][0]                          */
  double crop_y;       /* img_metas[0]['crop_offset'][1]                          */
  double scale;        /* img_metas[0].get('scale_factor', [1.0])[0]             */
  double org_w;        /* img_metas[0]['ori_shape'][1] (used only when flipped)   */
  int flip;            /* img_metas[0].get('flip', False)                         */
  int reserved;
} dfm_geometry_t;

/* ------------------------------------------------------------------------------------
 * DfMBackbone  (replaces mmdet3d/models/backbones/dfm_backbone.py:14-314:
 * build_dfm_cost + dres0/dres1 + hourglass + depth-pred convs + mono/stereo gate)
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_backbone dfm_backbone_t;

typedef struct dfm_backbone_desc {
  int in_channels;        /* DfMBackbone(in_channels=32)                       */
  int cv_channels;        /* cv_channels=32                                    */
  int feat_h, feat_w;     /* stereo feature size H x W (full image resolution) */
  int num_planes;         /* D = depth_cfg.num_bins / depth_cfg.downsample_factor */
  int cost_sample_factor; /* 4                                                 */
  int feat_sample_factor; /* 1                                                 */
  int conv_impl;          /* DFM_CONV_*                                        */
} dfm_backbone_desc_t;

int dfm_backbone_create(const dfm_backbone_desc_t* desc, dfm_backbone_t** out);
int dfm_backbone_destroy(dfm_backbone_t* bb);
/* Upload one parameter by its reference state_dict key (SURVEY.md 8a "State"), e.g.
 * "dres0.conv.weight" (32,64,3,3,3), "hg_stereo.0.conv5.0.weight" (ConvTranspose3d
 * layout in x out), "aggregate_cost.weight" (D,2D,1,1).  h_data: host fp32, reference
 * layout; the library repacks it for its kernels. */
int dfm_backbone_set_param(dfm_backbone_t* bb, const char* name, const float* h_data,
                           long long numel);
/* The injected attribute DfMBackbone.downsampled_depth (detectors/dfm.py:160-168). */
int dfm_backbone_set_depths(dfm_backbone_t* bb, const float* h_depths, int n);
/* Number of parameters still missing (0 = ready). */
int dfm_backbone_missing_params(const dfm_backbone_t* bb);
long long dfm_backbone_workspace_bytes(const dfm_backbone_t* bb);
/* DfMBackbone.forward (dfm_backbone.py:143-214), batch 1 (the reference supports
 * only B=1, :160).  d_cur/d_prev: [1,C,H,W] NCHW.  Outputs (any may be NULL):
 * d_cost [1,1,D,Ho,Wo], d_stereo / d_mono [1,32,D,Ho,Wo], NCDHW like the reference. */
int dfm_backbone_forward(dfm_backbone_t* bb, const float* d_cur, const float* d_prev,
                         const dfm_geometry_t* geom, float* d_cost, float* d_stereo,
                         float* d_mono, void* stream);
/* Same call for stereo features that are already channels-last [H][W][C] (what
 * dfm_stereo_tail_forward emits): skips the two NCHW -> NHWC transposes. */
int dfm_backbone_forward_cl(dfm_backbone_t* bb, const float* d_cur_cl, const float* d_prev_cl,
                            const dfm_geometry_t* geom, float* d_cost, float* d_stereo,
                            float* d_mono, void* stream);
/* Same call with HOST buffers: copies the two feature maps host->device, runs the
 * path, copies the outputs selected by out_flags (DFM_OUT_*) device->host, and
 * synchronises.  Buffers should be page-locked for full PCIe bandwidth. */
/* Optional: starts copying the NEXT pair host->device on a side stream and returns at once
 * (page-locked buffers).  A later dfm_backbone_forward_host with the same two host pointers
 * consumes the staged copy instead of copying again, so the transfer of pair i+1 overlaps the
 * processing of pair i.  Two pairs can be staged; the host buffers must stay unchanged until
 * the forward that consumes them returns. */
int dfm_backbone_prefetch_host(dfm_backbone_t* bb, const float* h_cur, const float* h_prev);
int dfm_backbone_forward_host(dfm_backbone_t* bb, const float* h_cur, const float* h_prev,
                              const dfm_geometry_t* geom, int out_flags, float* h_cost,
                              float* h_stereo, float* h_mono, void* stream);
/* Device pointer of the gated logits kept inside the handle after a forward
 * (lets a host-buffer caller chain dfm_depth_head_forward without a round trip). */
const float* dfm_backbone_cost_device(const dfm_backbone_t* bb);
/* Channels-last [D][Ho][Wo][cv] device copy of stereo_feat kept by the last forward (valid until
 * the next one): hand it to dfm_frustum_forward with DFM_LAYOUT_DHWC to skip a transpose. */
const float* dfm_backbone_stereo_feat_device(const dfm_backbone_t* bb);
/* Test hook: copies a named intermediate (channels-last [D][H][W][C]) to d_out.
 * Names: "raw0", "raw1", "c1".."c6", "p0", "logit", "cur" (cur_cost = cost0 + gn6(c6), the
 * input of the pred conv) and "cls3" (the cur-frame half's dres0 response on the first /
 * interior / last plane: [3][H][W][C]), with suffix "_mono" for the mono tower (which may
 * hold the z-shortened volume, see DESIGN.md).  Only the z-class first layer writes "cls3";
 * on that path the mono tower keeps dres0's output in "cls3_mono" and never writes
 * "raw0_mono".  A tensor the last forward did not write fails with DFM_ERR_STATE. */
int dfm_backbone_debug_tensor(dfm_backbone_t* bb, const char* name, float* d_out,
                              long long numel, void* stream);
/* Synchronises `stream` and reports asynchronous failures of this library's kernels
 * (CUDA errors, or an mbarrier hand-over that timed out inside a tensor-core kernel). */
int dfm_sync_check(void* stream);
/* Per-kernel device timing: when enabled, every conv launch is bracketed by CUDA events
 * on its own stream.  dfm_profile_report synchronises the device, writes one JSON object
 * {"<kernel class>": {"launches": n, "ms": total, "flops": algorithmic}, ...} into buf
 * (NUL-terminated, truncated to cap) and clears the record. */
int dfm_profile_enable(int on);
int dfm_profile_report(char* buf, int cap);
/* Counters since creation: kernels launched by this library / of which tensor-core. */
int dfm_launch_counters(long long* launches, long long* tc_launches);

/* ------------------------------------------------------------------------------------
 * build_dfm_cost alone (dfm_backbone.py:217-314), materialising the reference's
 * [1,2C,D,Ho,Wo] NCDHW volume.  Parity/bring-up op: the backbone never calls it (the
 * volume is consumed on the fly), tests use it to pin rows a1/a9 against the oracle.
 * h_depths: host [D].
 * ---------------------------------------------------------------------------------- */
int dfm_op_build_cost_volume(const float* d_cur, const float* d_prev, int C, int H, int W,
                             const float* h_depths, int D, int cost_sample_factor,
                             int feat_sample_factor, const dfm_geometry_t* geom,
                             float* d_volume, void* stream);

/* ------------------------------------------------------------------------------------
 * Generic 3x3x3 conv3d / conv_transpose3d building block (the cuDNN calls behind
 * models/utils/conv_modules.py:27-43,104-127 and mmcv ConvModule(Conv3d)).
 * d_x: NCDHW [1,Cin,Di,Hi,Wi]; h_w: host weight in the reference layout
 * ((Cout,Cin,3,3,3) or, transposed, (Cin,Cout,3,3,3)); d_y: NCDHW output.
 * stride/pad per (D,H,W); transposed uses stride 2, pad 1, output_padding 1.
 * ---------------------------------------------------------------------------------- */
int dfm_op_conv3d(const float* d_x, int Cin, int Di, int Hi, int Wi, const float* h_w,
                  int Cout, const int stride[3], const int pad[3], int transposed,
                  int conv_impl, float* d_y, void* stream);

/* ------------------------------------------------------------------------------------
 * DepthHead.forward with with_convs=False (mmdet3d/models/dense_heads/depth_head.py:
 * 190-212): x`factor` trilinear upsample (align_corners) -> softmax over depth ->
 * expectation over d_depth_samples [factor*D].  d_cost [1,1,D,Ho,Wo].
 * d_volume / d_softmax [1,1,fD,fHo,fWo] and d_preds [1,1,fHo,fWo]; any may be NULL
 * (skipping the two 4-D volumes is the fast path when only depth_preds is consumed).
 * ---------------------------------------------------------------------------------- */
int dfm_depth_head_forward(const float* d_cost, const float* d_depth_samples, int D, int Ho,
                           int Wo, int factor, float* d_volume, float* d_softmax,
                           float* d_preds, void* stream);

/* ------------------------------------------------------------------------------------
 * MultiViewDfM.feature_transformation lifting step (mmdet3d/models/detectors/
 * multiview_dfm.py:119-209 calling fusion_layers/point_fusion.py:14-106 with
 * aligned=False, valid_flag=True), one sample: nearest-tap gather of every voxel
 * centre into every (frame, view), valid-count averaging, temporal 'mean' or 'concat'.
 * d_feats [T*Nv, C, Hf, Wf]; h_lidar2img [T*Nv][16] row-major; the voxel-centre
 * coordinates per axis are passed in (the caller computes them exactly as
 * AlignedAnchor3DRangeGenerator does, core/anchor/anchor_3d_generator.py:283-310),
 * points are ordered z-major, then y, then x (the generator's permute at :327).  d_volume: [C*(concat?T:1), Nx, Ny, Nz].
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_lift_desc {
  int num_frames, num_views, channels, feat_h, feat_w;
  int n_voxels[3];            /* Nx, Ny, Nz                                  */
  float scale_x, scale_y;     /* img_meta['scale_factor'][:2]                */
  float crop_x, crop_y;       /* img_meta['img_crop_offset']                 */
  int flip;
  int input_h, input_w;       /* img_meta['input_shape']                     */
  int concat;                 /* temporal_aggregate == 'concat'              */
} dfm_lift_desc_t;
int dfm_multiview_lift(const dfm_lift_desc_t* desc, const float* d_feats,
                       const double* h_lidar2img, const int* h_img_w /* [T*Nv] img_shape w */,
                       const float* h_xs /* [Nx] */, const float* h_ys /* [Ny] */,
                       const float* h_zs /* [Nz] voxel-centre coordinates */,
                       float* d_volume, void* stream);
/* Same lifting, channels-last output [Nx][Ny][Nz][C*(concat?T:1)] -- the layout the necks' conv
 * loaders read (dfm_neck_forward_cl): the voxel's channels are one contiguous row, written by one
 * coalesced warp store, and the neck's NCDHW -> channels-last pass disappears.  Bit-identical
 * values.  (C == 64 and (concat or T == 1) run the fused kernel; other configurations run the
 * reference-layout kernel plus one transpose.) */
int dfm_multiview_lift_cl(const dfm_lift_desc_t* desc, const float* d_feats,
                          const double* h_lidar2img, const int* h_img_w, const float* h_xs,
                          const float* h_ys, const float* h_zs, float* d_volume_cl,
                          void* stream);
/* The same two liftings with the T*Nv views at separate addresses: h_view_feats is a host
 * array of T*Nv device pointers, each to one NCHW [C][Hf][Wf] view (current frame's views
 * first).  Values are bit-identical to the contiguous forms above, which build this table. */
int dfm_multiview_lift_views(const dfm_lift_desc_t* desc, const float* const* h_view_feats,
                             const double* h_lidar2img, const int* h_img_w, const float* h_xs,
                             const float* h_ys, const float* h_zs, float* d_volume,
                             void* stream);
int dfm_multiview_lift_views_cl(const dfm_lift_desc_t* desc, const float* const* h_view_feats,
                                const double* h_lidar2img, const int* h_img_w, const float* h_xs,
                                const float* h_ys, const float* h_zs, float* d_volume_cl,
                                void* stream);

/* ------------------------------------------------------------------------------------
 * DfMNeck / OutdoorImVoxelNeck, eval mode (mmdet3d/models/necks/dfm_neck.py:10-122,
 * imvoxel_neck.py:8-117): BatchNorm3d folded into per-channel affine.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_neck dfm_neck_t;
typedef struct dfm_neck_desc {
  int in_channels;  /* per-frame channels (64)                               */
  int out_channels; /* 256                                                   */
  int num_frames;   /* DfMNeck: stereo tower sees in_channels*num_frames; 0 => OutdoorImVoxelNeck */
  int nx, ny, nz;
  int conv_impl;
} dfm_neck_desc_t;
int dfm_neck_create(const dfm_neck_desc_t* desc, dfm_neck_t** out);
int dfm_neck_destroy(dfm_neck_t* neck);
/* Reference state_dict keys: "mono_layers.0.conv0.conv.weight", "...bn.weight/bias/
 * running_mean/running_var", "stereo_layers...", "aggregate_layer.weight"; for
 * OutdoorImVoxelNeck the prefix is "model.". */
int dfm_neck_set_param(dfm_neck_t* neck, const char* name, const float* h_data,
                       long long numel);
int dfm_neck_missing_params(const dfm_neck_t* neck);
/* d_x [1, Cin_total, Nx, Ny, Nz] -> d_bev [1, out_channels, Ny, Nx]. */
int dfm_neck_forward(dfm_neck_t* neck, const float* d_x, float* d_bev, void* stream);
/* d_x_cl: channels-last [Nx][Ny][Nz][C*T] (dfm_multiview_lift_cl's output) */
int dfm_neck_forward_cl(dfm_neck_t* neck, const float* d_x_cl, float* d_bev, void* stream);
/* Test hook: copies the raw (pre-BatchNorm) output of conv layer i of a tower, channels-last
 * [Nx][Ny][Zo][C], to d_out.  Names "mono.0" .. "mono.8" and "stereo.0" .. "stereo.8" (layer
 * order: res0.conv0, res0.conv1, down1, res2.conv0, res2.conv1, down3, res4.conv0, res4.conv1,
 * out5); OutdoorImVoxelNeck has only the "mono" tower.  A tensor the last forward did not write
 * fails with DFM_ERR_STATE, a numel other than the tensor's with DFM_ERR_INVALID. */
int dfm_neck_debug_tensor(dfm_neck_t* neck, const char* name, float* d_out, long long numel,
                          void* stream);

/* ------------------------------------------------------------------------------------
 * FrustumToVoxel (mmdet3d/models/necks/feature_transformation.py:12-173), the stage that
 * consumes the hot path's outputs (SURVEY.md section 8(f) row 1): the pseudo-lidar voxel grid
 * (detectors/dfm.py:174-211) is projected with cam2img[:3] (:175-187), stereo_feat / the depth
 * distribution / cur_sem_feats are grid-sampled there (:127-158), then voxel_convs
 * (Conv3d k3 + GroupNorm(32) + ReLU, :49-62) and AvgPool3d((4,1,1)) (:63,166).
 * ---------------------------------------------------------------------------------- */
#define DFM_LAYOUT_NCDHW 0 /* [C][D][H][W], the reference tensor layout   */
#define DFM_LAYOUT_DHWC 1  /* channels-last [D][H][W][C]                   */
typedef struct dfm_frustum dfm_frustum_t;
typedef struct dfm_frustum_desc {
  int num_3dconvs;       /* feature_transformation.py:17 (1..4)            */
  int cv_channels;       /* 32                                              */
  int out_channels;      /* 32                                              */
  int in_sem_channels;   /* 32                                              */
  int sem_atten_feat, stereo_atten_feat, cat_img_feature; /* :20-22        */
  int num_planes;        /* D of stereo_feat [1, cv, D, feat_h, feat_w]     */
  int feat_h, feat_w;
  int sem_h, sem_w;      /* cur_sem_feats [1, sem, sem_h, sem_w]            */
  int depth_factor;      /* softmax volume is [f*D][f*feat_h][f*feat_w]     */
  int nx, ny, nz;        /* voxel grid; coordinates_3d is [nz][ny][nx][3]   */
  float depth_min, depth_max; /* depth_cfg                                  */
  int conv_impl;         /* DFM_CONV_*                                      */
} dfm_frustum_desc_t;
/* h_xs [nx], h_ys [ny], h_zs [nz]: the separable pseudo-lidar voxel centres of
 * coordinates_3d (x = [0,0,:,0], y = [0,:,0,1], z = [:,0,0,2]). */
int dfm_frustum_create(const dfm_frustum_desc_t* desc, const float* h_xs, const float* h_ys,
                       const float* h_zs, dfm_frustum_t** out);
int dfm_frustum_destroy(dfm_frustum_t* f);
/* Reference state_dict keys: "voxel_convs.<i>.0.conv.weight", "voxel_convs.<i>.0.gn.weight",
 * "voxel_convs.<i>.0.gn.bias". */
int dfm_frustum_set_param(dfm_frustum_t* f, const char* name, const float* h_data,
                          long long numel);
int dfm_frustum_missing_params(const dfm_frustum_t* f);
/* One sample.  d_stereo_feat: device, layout as flagged.  The depth distribution is either the
 * materialised DepthHead output d_softmax [f*D][f*H][f*W] (the reference's argument) or, with
 * d_softmax == NULL, rebuilt on the fly from the low-res logits d_cost_logits [D][H][W]
 * (DfMBackbone's first output) so the 0.5-0.9 GB volume never exists; that pass is
 * DepthHead.forward's reduction, so with d_depth_samples [f*D] and d_depth_preds [f*H][f*W]
 * (both optional) it also returns the DepthHead's depth_preds and no separate
 * dfm_depth_head_forward call is needed.  d_sem: [sem][sem_h][sem_w] (NULL when
 * !cat_img_feature).  cam2img: 16 doubles, row-major img_meta['cam2img'].
 * pad_h/pad_w: img_metas[0]['pad_shape'].  d_out: [out_channels][nz/4][ny][nx]. */
int dfm_frustum_forward(dfm_frustum_t* f, const float* d_stereo_feat, int stereo_layout,
                        const float* d_softmax, const float* d_cost_logits,
                        const float* d_depth_samples, float* d_depth_preds, const float* d_sem,
                        const double* cam2img, int pad_h, int pad_w, float* d_out,
                        void* stream);
/* Test hook: copies "vox" (the gathered conv input, channels-last [nz][ny][nx][cv]) or "conv<i>"
 * (the raw output of voxel_convs[i], [nz][ny][nx][32]) to d_out.  The raw outputs share two
 * buffers, so "conv<i>" is gone once conv i + 2 ran: asking for it, or for a conv beyond
 * num_3dconvs, fails with DFM_ERR_STATE; a numel other than the tensor's with DFM_ERR_INVALID. */
int dfm_frustum_debug_tensor(dfm_frustum_t* f, const char* name, float* d_out, long long numel,
                             void* stream);

/* ------------------------------------------------------------------------------------
 * The hot-path segment of DfM.simple_test as one call with HOST buffers
 * (mmdet3d/models/detectors/dfm.py:296 `backbone_stereo(...)`, :420 `depth_head(...)`,
 * :423-425 `feature_transformation(...)`): (cur, prev) stereo features + cur semantic
 * features in, what the BEV stage consumes out -- voxel features [out][nz/4][ny][nx] and
 * DepthHead's depth_preds [fH][fW] (optionally the gated logits [D][Ho][Wo]).  Host->device
 * copies, the whole path and device->host copies run on `stream`; the call synchronises.
 * The pair may have been staged with dfm_backbone_prefetch_host.  stereo_feat never leaves
 * the device and the x4-upsampled DepthHead volumes are never built.  `fr` must have been
 * created for the backbone's volume shape (num_planes, feat_h = Ho, feat_w = Wo).
 * h_depth_samples: host [depth_factor * D] (DepthHead.depth_samples).
 * ---------------------------------------------------------------------------------- */
int dfm_pipeline_forward_host(dfm_backbone_t* bb, dfm_frustum_t* fr, const float* h_cur,
                              const float* h_prev, const float* h_sem,
                              const dfm_geometry_t* geom, const double* cam2img, int pad_h,
                              int pad_w, const float* h_depth_samples, float* h_voxel,
                              float* h_depth_preds, float* h_cost, void* stream);

/* ------------------------------------------------------------------------------------
 * The 2-D BEV stage behind FrustumToVoxel (SURVEY.md section 8(f) row 3; north_star's "3D box
 * regressions"): BEVHourglass (mmdet3d/models/backbones/bev_hourglass.py:11-137, GroupNorm
 * variant of configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:146-150) and LIGAAnchor3DHead's
 * forward (mmdet3d/models/dense_heads/liga_anchor3d_head.py:37-128).  All tensors NCHW fp32.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_bev_hourglass dfm_bev_hourglass_t;
typedef struct dfm_bev_desc {
  int in_channels;  /* 160 = 32 channels x 5 height slices (detectors/dfm.py:427-428) */
  int out_channels; /* 64                                                            */
  int ny, nx;       /* BEV grid, both multiples of 4 (304 x 288)                      */
  int conv_impl;    /* DFM_CONV_*                                                     */
} dfm_bev_desc_t;
int dfm_bev_hourglass_create(const dfm_bev_desc_t* desc, dfm_bev_hourglass_t** out);
int dfm_bev_hourglass_destroy(dfm_bev_hourglass_t* b);
/* Reference state_dict keys: "compress_conv.conv.weight", "compress_conv.gn.{weight,bias}",
 * "bev_hourglass.conv1.0.0.weight", "bev_hourglass.conv1.0.1.{weight,bias}",
 * "bev_hourglass.conv2.0.weight", ..., "bev_hourglass.conv5.0.weight" (ConvTranspose2d layout
 * in x out), "bev_hourglass.conv6.1.bias". */
int dfm_bev_hourglass_set_param(dfm_bev_hourglass_t* b, const char* name, const float* h_data,
                                long long numel);
int dfm_bev_hourglass_missing_params(const dfm_bev_hourglass_t* b);
/* BEVHourglass.forward (:39-50): d_x [in][ny][nx] -> d_prehg (optional) and d_out, both
 * [out][ny][nx] (spatial_features_2d_prehg, spatial_features_2d). */
int dfm_bev_hourglass_forward(dfm_bev_hourglass_t* b, const float* d_x, float* d_prehg,
                              float* d_out, void* stream);
/* Test hook: the raw output of "compress" or "conv1" .. "conv6", channels-last [H][W][C], as
 * the last forward wrote it (DFM_ERR_STATE otherwise; DFM_ERR_INVALID for a wrong numel). */
int dfm_bev_hourglass_debug_tensor(dfm_bev_hourglass_t* b, const char* name, float* d_out,
                                   long long numel, void* stream);

typedef struct dfm_anchor_head dfm_anchor_head_t;
typedef struct dfm_anchor_head_desc {
  int in_channels, feat_channels; /* 64, 64                                            */
  int num_convs;                  /* cls_convs / reg_convs depth (2)                   */
  int cls_channels;               /* num_anchors * num_classes      (18)               */
  int reg_channels;               /* num_anchors * box_code_size    (42)               */
  int dir_channels;               /* num_anchors * 2, 0 without direction classifier   */
  int ny, nx;
  int conv_impl;
} dfm_anchor_head_desc_t;
int dfm_anchor_head_create(const dfm_anchor_head_desc_t* desc, dfm_anchor_head_t** out);
int dfm_anchor_head_destroy(dfm_anchor_head_t* h);
/* Keys: "cls_convs.<i>.conv.weight", "cls_convs.<i>.gn.{weight,bias}", "reg_convs.<i>...",
 * "conv_cls.{weight,bias}", "conv_reg.{weight,bias}", "conv_dir_cls.{weight,bias}". */
int dfm_anchor_head_set_param(dfm_anchor_head_t* h, const char* name, const float* h_data,
                              long long numel);
int dfm_anchor_head_missing_params(const dfm_anchor_head_t* h);
/* LIGAAnchor3DHead.forward_single (:108-128): d_x [64][ny][nx] -> cls_score
 * [cls_channels][ny][nx], bbox_pred [reg_channels][ny][nx], dir_cls_preds
 * [dir_channels][ny][nx]. */
int dfm_anchor_head_forward(dfm_anchor_head_t* h, const float* d_x, float* d_cls, float* d_bbox,
                            float* d_dir, void* stream);
/* Test hook: the raw output, channels-last [ny][nx][C], of "cls<i>" / "reg<i>" (i < num_convs)
 * or of the output convs "cls_out" (conv_cls + conv_dir_cls, C = cls + dir channels padded to
 * a multiple of 32) and "reg_out" (C = reg channels padded likewise), without bias.  A tensor
 * the last forward did not write fails with DFM_ERR_STATE, a wrong numel with DFM_ERR_INVALID. */
int dfm_anchor_head_debug_tensor(dfm_anchor_head_t* h, const char* name, float* d_out,
                                 long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * Anchor3DHead's forward (mmdet3d/models/dense_heads/anchor3d_head.py:139-164), the box head
 * of both MultiViewDfM (Waymo) configs: three 1x1 convs with bias on the BEV map that
 * DfMNeck / OutdoorImVoxelNeck return.  All tensors NCHW fp32.  conv_impl AUTO / TC run the
 * three convs as one wgmma GEMM when feat_channels % 16 == 0 and the shape fits the kernel
 * (combined output channels <= 128 and its shared-memory image); SIMT, and AUTO on other
 * shapes, run the fp32 CUDA-core 2-D conv; TC on a shape without the kernel fails at create
 * with DFM_ERR_INVALID.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_anchor3d_head dfm_anchor3d_head_t;
typedef struct dfm_anchor3d_head_desc {
  int feat_channels;  /* input channels of the three convs (256)                       */
  int cls_channels;   /* num_anchors * num_classes (18)                               */
  int reg_channels;   /* num_anchors * box_code_size (42)                             */
  int dir_channels;   /* num_anchors * 2 (12), 0 without direction classifier         */
  int ny, nx;         /* BEV grid (300 x 220)                                         */
  int conv_impl;      /* DFM_CONV_AUTO / DFM_CONV_SIMT / DFM_CONV_TC                  */
} dfm_anchor3d_head_desc_t;
int dfm_anchor3d_head_create(const dfm_anchor3d_head_desc_t* desc, dfm_anchor3d_head_t** out);
int dfm_anchor3d_head_destroy(dfm_anchor3d_head_t* h);
/* Keys: "conv_cls.{weight,bias}", "conv_reg.{weight,bias}", "conv_dir_cls.{weight,bias}"
 * (weights (out, feat_channels, 1, 1)); a wrong numel fails with DFM_ERR_INVALID. */
int dfm_anchor3d_head_set_param(dfm_anchor3d_head_t* h, const char* name, const float* h_data,
                                long long numel);
int dfm_anchor3d_head_missing_params(const dfm_anchor3d_head_t* h);
/* forward_single: d_x [feat_channels][ny][nx] -> cls_score [cls_channels][ny][nx], bbox_pred
 * [reg_channels][ny][nx], dir_cls_preds [dir_channels][ny][nx] (d_dir may be NULL when
 * dir_channels == 0).  DFM_ERR_STATE while a parameter is missing. */
int dfm_anchor3d_head_forward(dfm_anchor3d_head_t* h, const float* d_x, float* d_cls,
                              float* d_bbox, float* d_dir, void* stream);

/* ------------------------------------------------------------------------------------
 * voxel_sample (mmdet3d/models/fusion_layers/point_fusion.py:324-410): frustum-from-voxel
 * resampling for an optional depth head of MultiViewDfM (detectors/multiview_dfm.py:220-256;
 * no shipped config enables it).  d_voxel [C][Nx][Ny][Nz] -> d_out [C][num_depths][out_h][out_w],
 * out_h/out_w = round(img_pad_shape / downsample_factor); h_depths: host [num_depths] =
 * depth_samples[::downsample_factor]; h_proj: 16 doubles, the (lidar/cam)2img matrix.
 * grid_sample semantics: zeros padding, align_corners=True, trilinear (aligned) or nearest.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_voxel_sample_desc {
  int channels, nx, ny, nz;
  float voxel_range[6];
  float voxel_size[3];
  int num_depths, out_h, out_w, downsample_factor;
  float scale_x, scale_y;  /* img_scale_factor */
  float crop_x, crop_y;    /* img_crop_offset  */
  int flip, img_w;         /* img_flip, img_shape[1] */
  int aligned;             /* 1: trilinear, 0: nearest */
} dfm_voxel_sample_desc_t;
int dfm_voxel_sample(const dfm_voxel_sample_desc_t* desc, const float* d_voxel,
                     const float* h_depths, const double* h_proj, float* d_out, void* stream);

/* Asynchronous form of the same call: submit enqueues the host->device copies, the path and
 * the device->host copies of the outputs (those on a side stream, so they overlap the NEXT
 * frame's compute) and returns at once; dfm_pipeline_wait blocks until the outputs of the
 * oldest submitted frame are in host memory and reports asynchronous failures.  At most two
 * frames may be in flight; host input buffers must stay unchanged until the wait for their
 * frame returns, output buffers must not be read before it. */
int dfm_pipeline_submit_host(dfm_backbone_t* bb, dfm_frustum_t* fr, const float* h_cur,
                             const float* h_prev, const float* h_sem,
                             const dfm_geometry_t* geom, const double* cam2img, int pad_h,
                             int pad_w, const float* h_depth_samples, float* h_voxel,
                             float* h_depth_preds, void* stream);
int dfm_pipeline_wait(dfm_backbone_t* bb);
/* dfm_backbone_prefetch_host for the pipeline: also stages the NEXT frame's sem features
 * (`sem_numel` floats, may be NULL / 0) together with its pair on the side stream.  A small
 * host->device copy issued at submit time would queue on the copy engine behind this bulk
 * copy and stall the compute stream, so everything a frame reads
 * from the host should be handed over here, one frame ahead. */
int dfm_pipeline_prefetch_host(dfm_backbone_t* bb, const float* h_cur, const float* h_prev,
                               const float* h_sem, long long sem_numel);

/* ------------------------------------------------------------------------------------
 * The tail of SPPUNetNeck (mmdet3d/models/necks/spp_unet_neck.py:60-75 `lastconv`, applied at
 * :110; SURVEY.md section 8(f) row 2): Conv2d 3x3 (32->32) + GroupNorm(32) + ReLU + Conv2d 1x1
 * (32->32, no bias) producing the full-resolution stereo feature that build_dfm_cost samples.
 * d_x [32][H][W] (the up-convolved feature, NCHW) -> d_out_cl [H][W][32] channels-last (feed it
 * to dfm_backbone_forward_cl) and / or d_out_nchw [32][H][W] (the reference's return value).
 * Keys: "lastconv.0.conv.weight" (32,32,3,3), "lastconv.0.gn.weight", "lastconv.0.gn.bias",
 * "lastconv.1.weight" (32,32,1,1).
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_stereo_tail dfm_stereo_tail_t;
int dfm_stereo_tail_create(int H, int W, int conv_impl, dfm_stereo_tail_t** out);
int dfm_stereo_tail_destroy(dfm_stereo_tail_t* t);
int dfm_stereo_tail_set_param(dfm_stereo_tail_t* t, const char* name, const float* h_data,
                              long long numel);
int dfm_stereo_tail_missing_params(const dfm_stereo_tail_t* t);
int dfm_stereo_tail_forward(dfm_stereo_tail_t* t, const float* d_x, float* d_out_cl,
                            float* d_out_nchw, void* stream);

/* ------------------------------------------------------------------------------------
 * The whole SPPUNetNeck of the shipped KITTI config (mmdet3d/models/necks/spp_unet_neck.py;
 * configs/dfm/dfm_r34_1x8_kitti-3d-3class.py `neck`: in_channels [3, 64, 128, 128, 128],
 * start_level 2, spp_channel 32, with_upconv, cat_img_feature, GN(32)), one image per call.
 * H x W is the image size: d_img [3][H][W], d_f1 [64][H/2][W/2], d_f2 / d_f3 / d_f4
 * [128][H/4][W/4], all NCHW.  Outputs: stereo_feature as d_stereo_cl [H][W][32] (channels-last,
 * for dfm_backbone_forward_cl) and / or d_stereo_nchw [32][H][W]; sem_feature d_sem
 * [32][H/4][W/4] NCHW (required).
 * create: H and W multiples of 4, and floor(H/256) * floor(W/256) >= 2 (the reference's
 * GroupNorm of the 64x64 SPP branch needs two cells); else DFM_ERR_INVALID.
 * Keys: the reference state_dict without num_batches_tracked (42 entries): spp_branches.{0..3}.1.
 * {conv.weight, gn.weight, gn.bias}, upconv_module.{conv,redir}.{0,1}.0.weight and .1.{weight,
 * bias, running_mean, running_var} (BatchNorm, folded), lastconv.*, rpnconv.{0,1}.{conv.weight,
 * gn.weight, gn.bias}.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_spp_neck dfm_spp_neck_t;
int dfm_spp_neck_create(int H, int W, int conv_impl, dfm_spp_neck_t** out);
int dfm_spp_neck_destroy(dfm_spp_neck_t* n);
int dfm_spp_neck_set_param(dfm_spp_neck_t* n, const char* name, const float* h_data,
                           long long numel);
int dfm_spp_neck_missing_params(const dfm_spp_neck_t* n);
int dfm_spp_neck_forward(dfm_spp_neck_t* n, const float* d_img, const float* d_f1,
                         const float* d_f2, const float* d_f3, const float* d_f4,
                         float* d_stereo_cl, float* d_stereo_nchw, float* d_sem, void* stream);
/* Test hook: channels-last copy of an intermediate of the last forward.  Names: the raw conv
 * outputs "conv0" (upconv.conv.0, [H/4][W/4][64]), "redir0" ([H/2][W/2][64]), "conv1"
 * ([H/2][W/2][32]), "rpn0" ([H/4][W/4][128]), "rpn1" ([H/4][W/4][32]), "lastconv" ([H][W][32]);
 * the pooled f4 "pool64" .. "pool8" ([Ph][Pw][128]); the branch maps before upsampling
 * "spp64" .. "spp8" ([Ph][Pw][32], after GroupNorm + ReLU); "concat" ([H/4][W/4][512]); "x0"
 * ([H/2][W/2][64]); "x1" ([H][W][32]).  DFM_ERR_STATE if the last forward did not write it,
 * DFM_ERR_INVALID on a wrong element count. */
int dfm_spp_neck_debug_tensor(dfm_spp_neck_t* n, const char* name, float* d_out,
                              long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * mmdet's FPN image neck as both MultiViewDfM (Waymo) configs use it (`neck`: in_channels
 * [256, 512, 1024, 2048], out_channels 64, num_outs 4; start_level 0, no extra convs, no norm,
 * no activation, nearest upsampling to the finer level's size), for num_images images per
 * call.  merged_3 = lateral_3(x_3); merged_l = lateral_l(x_l) + up(merged_{l+1});
 * out_l = fpn_conv_l(merged_l).  The lateral 1x1 convs run as one wgmma GEMM per level with
 * the merge in its epilogue when out_channels == 64 (conv_impl AUTO / TC); SIMT, and AUTO with
 * out_channels == 32, run them on fp32 CUDA cores.  TC with out_channels != 64 fails at
 * create with DFM_ERR_INVALID, as do channel counts that are not multiples of 16, other
 * out_channels, and levels with in_channels * h * w >= 2^31.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_fpn dfm_fpn_t;
typedef struct dfm_fpn_desc {
  int in_channels[4];  /* channels of C2..C5 (256, 512, 1024, 2048)                       */
  int out_channels;    /* 64 (tensor cores) or 32                                         */
  int level_h[4];      /* sizes of the four levels, finest first (208, 104, 52, 26)      */
  int level_w[4];      /* (312, 156, 78, 39)                                              */
  int num_images;      /* images per call (views x frames of a sample)                   */
  int conv_impl;       /* DFM_CONV_AUTO / DFM_CONV_SIMT / DFM_CONV_TC                     */
} dfm_fpn_desc_t;
int dfm_fpn_create(const dfm_fpn_desc_t* desc, dfm_fpn_t** out);
int dfm_fpn_destroy(dfm_fpn_t* f);
/* Sets the number of images the next forwards take, keeping the handle and its parameters
 * (buffers grow at the next forward when needed).  DFM_ERR_INVALID when num_images < 1 or the
 * batch exceeds the limits create checks. */
int dfm_fpn_set_num_images(dfm_fpn_t* f, int num_images);
/* Keys: "lateral_convs.{0..3}.conv.{weight,bias}" (weights (out, in_l, 1, 1)) and
 * "fpn_convs.{0..3}.conv.{weight,bias}" (weights (out, out, 3, 3)); a wrong numel fails with
 * DFM_ERR_INVALID. */
int dfm_fpn_set_param(dfm_fpn_t* f, const char* name, const float* h_data, long long numel);
int dfm_fpn_missing_params(const dfm_fpn_t* f);
/* d_in[l]: [num_images][in_channels[l]][level_h[l]][level_w[l]] NCHW -> d_out[l]:
 * [num_images][out_channels][level_h[l]][level_w[l]] NCHW.  DFM_ERR_STATE while a parameter
 * is missing. */
int dfm_fpn_forward(dfm_fpn_t* f, const float* const* d_in, float* const* d_out, void* stream);
/* Test hook: channels-last copy of an intermediate of the last forward.  "merged0" ..
 * "merged3": the merged laterals [num_images][h_l][w_l][out_channels]; "fpn0" .. "fpn3": the
 * raw fpn_conv outputs before the bias, same layout.  DFM_ERR_STATE if the last forward did
 * not write it, DFM_ERR_INVALID on a wrong element count. */
int dfm_fpn_debug_tensor(dfm_fpn_t* f, const char* name, float* d_out, long long numel,
                         void* stream);

/* ------------------------------------------------------------------------------------
 * DfM's LIGAResNet-34 image backbone as the shipped KITTI config builds it (`backbone`:
 * depth 34, strides (1, 2, 1, 1), dilations (1, 1, 2, 4), num_channels_factor (1, 2, 2, 2),
 * no max-pool, no ReLU after the residual add, BatchNorm in eval form), for num_images images
 * per call.  Stem 7x7 / 2 (3 -> 64); layer1: 3 blocks at 64 channels, H2 = ceil(H / 2);
 * layer2: 4 blocks at 128 channels, the first with stride 2 and a 1x1 / 2 downsample,
 * H4 = ceil(H2 / 2); layer3: 6 blocks, dilation 2; layer4: 3 blocks, dilation 4.
 * AUTO / TC run every 3x3 stride-1 conv on the wgmma implicit-GEMM kernel and the stem, the
 * stride-2 conv and the downsample on fp32 CUDA cores; SIMT runs every conv on fp32 CUDA
 * cores.  Fails at create with DFM_ERR_INVALID on an empty image or num_images < 1.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_liga_resnet dfm_liga_resnet_t;
typedef struct dfm_liga_resnet_desc {
  int height;          /* image size H x W (384 x 1248 in the KITTI test pipeline)        */
  int width;
  int num_images;      /* images per call (cur + prev of a frame: 2)                      */
  int conv_impl;       /* DFM_CONV_AUTO / DFM_CONV_SIMT / DFM_CONV_TC                     */
} dfm_liga_resnet_desc_t;
int dfm_liga_resnet_create(const dfm_liga_resnet_desc_t* desc, dfm_liga_resnet_t** out);
int dfm_liga_resnet_destroy(dfm_liga_resnet_t* r);
/* Sets the number of images the next forwards take, keeping the handle and its parameters
 * (buffers grow at the next forward when needed).  DFM_ERR_INVALID when num_images < 1 or the
 * batch exceeds the limits create checks. */
int dfm_liga_resnet_set_num_images(dfm_liga_resnet_t* r, int num_images);
/* Keys are the reference state_dict's: "conv1.weight", "bn1.{weight,bias,running_mean,
 * running_var}", "layer{1..4}.{j}.conv{1,2}.weight", "layer{1..4}.{j}.bn{1,2}.*",
 * "layer2.0.downsample.0.weight", "layer2.0.downsample.1.*" ("num_batches_tracked" is not
 * needed); a wrong numel fails with DFM_ERR_INVALID. */
int dfm_liga_resnet_set_param(dfm_liga_resnet_t* r, const char* name, const float* h_data,
                              long long numel);
int dfm_liga_resnet_missing_params(const dfm_liga_resnet_t* r);
/* d_img: [num_images][3][H][W] NCHW -> d_out[0]: [num_images][64][H2][W2], d_out[1..3]:
 * [num_images][128][H4][W4], NCHW.  DFM_ERR_STATE while a parameter is missing. */
int dfm_liga_resnet_forward(dfm_liga_resnet_t* r, const float* d_img, float* const* d_out,
                            void* stream);
/* Test hook: channels-last [num_images][h][w][C] copy of an intermediate of the last forward:
 * "stem" (raw conv1 output), "layerI.J.conv1" / "layerI.J.conv2" / "layer2.0.downsample" (raw
 * conv outputs, before BatchNorm), "layerI.J" (block outputs).  DFM_ERR_STATE if the last
 * forward did not write it, DFM_ERR_INVALID on a wrong element count. */
int dfm_liga_resnet_debug_tensor(dfm_liga_resnet_t* r, const char* name, float* d_out,
                                 long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * mmdet's ResNet-101 with DCNv2 as both MultiViewDfM (Waymo) configs build it (`backbone`:
 * depth 101, style pytorch, BatchNorm in eval form, dcn DCNv2 with deform_groups 1 and
 * fallback_on_stride False in layer3 / layer4), for num_images images per call.  Stem 7x7 / 2
 * (3 -> 64), BN, ReLU, max-pool 3x3 / 2 / 1; Bottleneck stages of 3, 4, 23, 3 blocks at
 * 256, 512, 1024, 2048 output channels; H_l = ceil(H_{l-1} / 2) at every stride-2 step.  The
 * conv2 of layer3 / layer4 is a modulated deformable conv whose offsets and masks come from its
 * conv_offset (3x3, 27 channels, bias).  AUTO / TC run every conv but the stem on wgmma kernels;
 * SIMT runs every conv on fp32 CUDA cores.  Fails at create with DFM_ERR_INVALID on an empty
 * image, num_images < 1 or num_images * ceil(H / 2) * ceil(W / 2) >= 2^31.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_resnet101 dfm_resnet101_t;
typedef struct dfm_resnet101_desc {
  int height;          /* image size H x W (832 x 1248 in the Waymo test pipeline)         */
  int width;
  int num_images;      /* images per call (views x frames of a sample)                    */
  int conv_impl;       /* DFM_CONV_AUTO / DFM_CONV_SIMT / DFM_CONV_TC                     */
} dfm_resnet101_desc_t;
int dfm_resnet101_create(const dfm_resnet101_desc_t* desc, dfm_resnet101_t** out);
int dfm_resnet101_destroy(dfm_resnet101_t* r);
/* Sets the number of images the next forwards take, keeping the handle and its parameters
 * (buffers grow at the next forward when needed).  DFM_ERR_INVALID when num_images < 1 or the
 * batch exceeds the limits create checks. */
int dfm_resnet101_set_num_images(dfm_resnet101_t* r, int num_images);
/* Keys are mmdet's state_dict's: "conv1.weight", "bn1.{weight,bias,running_mean,running_var}",
 * "layer{1..4}.{j}.conv{1,2,3}.weight", "layer{1..4}.{j}.bn{1,2,3}.*",
 * "layer{3,4}.{j}.conv2.conv_offset.{weight,bias}", "layer{1..4}.0.downsample.0.weight",
 * "layer{1..4}.0.downsample.1.*" ("num_batches_tracked" is not needed); a wrong numel fails
 * with DFM_ERR_INVALID. */
int dfm_resnet101_set_param(dfm_resnet101_t* r, const char* name, const float* h_data,
                            long long numel);
int dfm_resnet101_missing_params(const dfm_resnet101_t* r);
/* d_img: [num_images][3][H][W] NCHW -> d_out[l]: [num_images][256 << l][H_{l+2}][W_{l+2}]
 * NCHW (H_2 = H / 4 .. H_5 = H / 32, rounded up).  DFM_ERR_STATE while a parameter is
 * missing. */
int dfm_resnet101_forward(dfm_resnet101_t* r, const float* d_img, float* const* d_out,
                          void* stream);
/* Test hook: channels-last [num_images][h][w][C] copy of an intermediate of the last forward:
 * "stem" (raw conv1 output), "pool" (the max-pooled activation), "layerI.J.conv{1,2,3}" and
 * "layerI.0.downsample" (raw conv outputs, before BatchNorm), "layerI.J.conv2.conv_offset"
 * (conv_offset + bias, 27 channels padded to 32), "layerI.J.conv2.offset_mask" (the same with
 * the sigmoid applied to channels 18..26: what the deformable conv reads), "layerI.J" (block
 * outputs).  DFM_ERR_STATE if the last forward did not write it, DFM_ERR_INVALID on a wrong
 * element count. */
int dfm_resnet101_debug_tensor(dfm_resnet101_t* r, const char* name, float* d_out,
                               long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * get_bboxes of Anchor3DHead and LIGAAnchor3DHead (one feature level) for `batch` samples per
 * call: class scores (sigmoid, or softmax with the background column last), the top nms_pre
 * anchors by their best class score (skipped when the grid has no more than nms_pre anchors),
 * DeltaXYZWLHRBBoxCoder decode, per-class score_thr filter and rotated BEV NMS, the cut to
 * max_num by score, and the direction-classifier yaw fix.  Anchor index (y * nx + x) *
 * num_anchors + j; class channel j * ncol + c, box channel j * 7 + k, direction channel
 * j * 2 + k.  No host synchronisation inside forward.  Create fails with DFM_ERR_INVALID when a
 * class could receive more than 4096 NMS candidates (min(nms_pre, anchors), or all anchors when
 * nms_pre <= 0) or num_classes > 16.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_box_post dfm_box_post_t;
typedef struct dfm_box_post_desc {
  int num_classes;        /* C foreground classes                                          */
  int num_anchors;        /* anchors per cell (sizes x rotations), 6 in the shipped configs */
  int ny;                 /* feature map H                                                 */
  int nx;                 /* feature map W                                                 */
  int batch;              /* samples per call                                              */
  int use_sigmoid;        /* 1: C sigmoid columns; 0: C + 1 softmax columns               */
  int nms_pre;            /* test_cfg.nms_pre (<= 0: no pre-NMS top-k)                    */
  int max_num;            /* test_cfg.max_num                                              */
  float score_thr;        /* test_cfg.score_thr (strict, in fp32)                          */
  float nms_thr;          /* test_cfg.nms_thr (a box is suppressed when IoU > nms_thr)     */
  float dir_offset;       /* head dir_offset                                               */
  float dir_limit_offset; /* head dir_limit_offset                                         */
} dfm_box_post_desc_t;
/* h_anchors: host [ny * nx * num_anchors][7] fp32 (x, y, z, w, l, h, yaw), copied at create. */
int dfm_box_post_create(const dfm_box_post_desc_t* desc, const float* h_anchors,
                        dfm_box_post_t** out);
int dfm_box_post_destroy(dfm_box_post_t* h);
/* d_cls [batch][num_anchors * ncol][ny][nx], d_bbox [batch][num_anchors * 7][ny][nx],
 * d_dir [batch][num_anchors * 2][ny][nx] (NCHW) -> d_boxes [batch][max_num][7],
 * d_scores [batch][max_num], d_labels [batch][max_num] (int32), d_count [batch].  Entries
 * at and past d_count[b] are not written. */
int dfm_box_post_forward(dfm_box_post_t* h, const float* d_cls, const float* d_bbox,
                         const float* d_dir, float* d_boxes, float* d_scores, int* d_labels,
                         int* d_count, void* stream);
/* Test hook: int32 [batch][K] (K = anchors that enter decoding) from the last forward:
 * "topk_index" (selected anchors by score descending, anchor index ascending; DFM_ERR_STATE
 * when the grid skipped the top-k), "cls<c>_candidates" (anchors passing score_thr for class c,
 * in NMS processing order), "cls<c>_keep" (anchors kept by class c's NMS, in order); -1 past
 * each sample's count.  DFM_ERR_INVALID on a wrong element count. */
int dfm_box_post_debug_tensor(dfm_box_post_t* h, const char* name, int* d_out, long long numel,
                              void* stream);
/* Test hook: the fp32 rotated IoU the NMS of dfm_box_post_forward decides with, pair by pair.
 * d_a, d_b: device [n][5] (x, y, w, h, yaw), the NMS box of the earlier and of the later
 * candidate; d_iou: device [n].  DFM_ERR_INVALID on n <= 0 or a null pointer. */
int dfm_op_rotated_iou(const float* d_a, const float* d_b, int n, float* d_iou, void* stream);

/* ------------------------------------------------------------------------------------
 * Training losses of Anchor3DHead and LIGAAnchor3DHead (one feature level) for `batch` samples
 * per call: MaxIoUAssigner on the nearest-BEV IoU (one assigner per anchor size), PseudoSampler,
 * DeltaXYZWLHRBBoxCoder targets and direction targets, then the sigmoid focal loss, SmoothL1
 * (with the sin difference on the yaw channel when diff_rad_by_sin), the direction softmax
 * cross-entropy and, for LIGA with loss_iou, 1 - IoU3D of the decoded positives.  Anchor index
 * (y * nx + x) * A + s * num_rotations + r, A = num_sizes * num_rotations; class channel
 * j * num_classes + c, box channel j * 7 + k, direction channel j * 2 + k (NCHW).  No host
 * synchronisation inside forward or finish; sums run in a fixed order, so repeated calls are
 * bitwise equal.  Create fails with DFM_ERR_INVALID on more than 16 classes or 8 sizes.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_anchor_loss dfm_anchor_loss_t;
typedef struct dfm_anchor_loss_desc {
  int num_classes;              /* C sigmoid classes                                          */
  int num_sizes;                /* anchor sizes, one assigner each                            */
  int num_rotations;            /* rotations per size                                         */
  int ny, nx, batch;            /* feature map and samples per call                           */
  int assign_per_class;         /* 1: size s sees only GT of label s; 0: every GT             */
  int diff_rad_by_sin;          /* 1: yaw channel as sin(p)cos(t) against cos(p)sin(t)        */
  int use_direction_classifier; /* 1: direction loss                                          */
  int with_iou;                 /* 1: 1 - IoU3D term (LIGA loss_iou)                          */
  int liga;                     /* normalisers: 0 Anchor3DHead, 1 LIGAAnchor3DHead             */
  float pos_iou_thr[8];         /* per assigner                                               */
  float neg_iou_thr[8];
  float min_pos_iou[8];
  float pos_weight;             /* train_cfg.pos_weight (<= 0: 1)                              */
  float gamma, alpha;           /* FocalLoss                                                  */
  float beta;                   /* SmoothL1Loss                                               */
  float loss_weight[4];         /* cls, bbox, dir, iou                                        */
  float dir_offset, dir_limit_offset;
  float normalizer_clamp_value; /* LIGA                                                       */
} dfm_anchor_loss_desc_t;
/* h_anchors: host [ny * nx * A][7] fp32, copied at create. */
int dfm_anchor_loss_create(const dfm_anchor_loss_desc_t* desc, const float* h_anchors,
                           dfm_anchor_loss_t** out);
int dfm_anchor_loss_destroy(dfm_anchor_loss_t* h);
/* d_cls [batch][A * C][ny][nx], d_bbox [batch][A * 7][ny][nx], d_dir [batch][A * 2][ny][nx];
 * GT packed: d_gt_boxes [G][7] LiDAR boxes, d_gt_labels [G] int32 in 0..C-1, d_gt_off /
 * h_gt_off [batch + 1] on the device and the host (at most 1024 boxes per sample).  Writes the
 * gradients of the unnormalised, unweighted loss sums into each non-null d_grad_* (same layouts
 * as the inputs; d_grad_iou is the IoU term's gradient with respect to d_bbox, only with
 * with_iou) and d_norm [1] = sum over samples of max(positives, 1).  A GT label outside
 * 0..C-1 is detected on the device and makes every loss of the next finish NaN.  Where a decoded
 * target value is NaN the IoU term uses the prediction's value instead (iou3d_loss); its
 * gradient then flows through the prediction's side of the IoU only, not also through the
 * substituted target value as the reference's autograd does.  Such targets come only from
 * degenerate GT (a size <= 0 or a non-finite value). */
int dfm_anchor_loss_forward(dfm_anchor_loss_t* h, const float* d_cls, const float* d_bbox,
                            const float* d_dir, const float* d_gt_boxes, const int* d_gt_labels,
                            const int* d_gt_off, const int* h_gt_off, float* d_grad_cls,
                            float* d_grad_bbox, float* d_grad_dir, float* d_grad_iou,
                            float* d_norm, void* stream);
/* From the last forward and d_avg [1] (the normaliser: d_norm, or its all-reduced mean for
 * LIGA): d_losses [4] (cls, bbox, dir, iou) and d_scales [4], the factor each stored gradient
 * takes to become that of its loss. */
int dfm_anchor_loss_finish(dfm_anchor_loss_t* h, const float* d_avg, float* d_losses,
                           float* d_scales, void* stream);
/* Test hook, from the last forward, [batch][N] per anchor: "assigned_gt" int32 (-1 ignored,
 * 0 negative, g + 1 for the sample's GT g), "labels" int32 (C for negatives and ignored),
 * "label_weights" fp32, "dir_targets" int32, "bbox_targets" fp32 [batch][N][7].
 * DFM_ERR_STATE before a forward, DFM_ERR_INVALID on an unknown name or wrong element count. */
int dfm_anchor_loss_debug_tensor(dfm_anchor_loss_t* h, const char* name, void* d_out,
                                 long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * Training loss of DfM's 2-D auxiliary LIGAATSSHead (liga_atss_head.py:176-270, 380-483 with
 * mmdet 2.x's ATSSHead.loss) for `batch` images of num_levels levels per call, one square anchor
 * of side octave_base_scale * stride per location (AnchorGenerator, ratios [1], one scale,
 * centre offset 0): ATSS3DCenterAssigner (topk nearest valid anchors per level to the GT's
 * projected 3-D centre, IoU >= mean + std of the candidates, anchor centre more than 0.01 inside
 * the 2-D box, highest IoU wins), PseudoSampler, DeltaXYWHBBoxCoder targets (means 0) and
 * centerness targets, then per level the sigmoid focal loss, GIoU of the decoded positives
 * weighted by their centerness targets, and the centerness BCE.  Anchors of level l at
 * (x * stride, y * stride), index off_l + y * feat_w + x; the valid anchors of each image come
 * from its pad shape (min(ceil(pad / stride), feat) rows and columns).  Two orders the
 * reference leaves to torch are fixed: equal distances at the topk-th candidate keep the lower
 * anchor index, and an anchor positive for several GT with equal IoU goes to the first GT.  The
 * threshold's mean and std are formed in fp64 in candidate order (level, then distance), each
 * rounded to fp32, then added in fp32.  No host synchronisation inside forward or finish; sums
 * run in a fixed order, so repeated calls are bitwise equal.  Create fails with DFM_ERR_INVALID
 * on more than 16 classes, 8 levels or 32 images, or topk other than 9.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_atss_loss dfm_atss_loss_t;
typedef struct dfm_atss_loss_desc {
  int num_classes;              /* C sigmoid classes                                          */
  int num_levels;               /* L                                                          */
  int strides[8];               /* per level, integer                                         */
  int feat_h[8], feat_w[8];     /* per level                                                  */
  int batch;                    /* images per call                                            */
  int topk;                     /* ATSS3DCenterAssigner topk (9)                              */
  float octave_base_scale;      /* anchor side / stride                                       */
  float target_stds[4];         /* DeltaXYWHBBoxCoder; x = y and w = h                        */
  float wh_ratio_clip;          /* size deltas clamped to +- |log(wh_ratio_clip)|             */
  float giou_eps;               /* GIoULoss eps                                               */
  float gamma, alpha;           /* FocalLoss                                                  */
  float loss_weight[3];         /* cls, bbox, centerness                                      */
} dfm_atss_loss_desc_t;
int dfm_atss_loss_create(const dfm_atss_loss_desc_t* desc, dfm_atss_loss_t** out);
int dfm_atss_loss_destroy(dfm_atss_loss_t* h);
/* d_cls / d_bbox / d_centerness: host arrays of num_levels device pointers, level l
 * [batch][C][feat_h][feat_w], [batch][4 * C][feat_h][feat_w] (channel k * C + c: coordinate k of
 * class c) and [batch][1][feat_h][feat_w].  GT packed: d_gt_boxes [G][6] (2-D box x1, y1, x2, y2,
 * then the projected 3-D centre x, y), d_gt_labels [G] int32 in 0..C-1, d_gt_off / h_gt_off
 * [batch + 1] on the device and the host; h_pad_shape [batch][2] (pad height, width) on the host.
 * Writes the gradients of the unnormalised, unweighted per-level sums into each non-null entry of
 * the host arrays d_grad_* (the arrays themselves may be NULL; same layouts as the inputs) and
 * d_norm [2] = (sum over images of max(positives, 1), sum of the centerness targets).  A GT
 * label outside 0..C-1 is detected on the device and makes every loss of the next finish NaN. */
int dfm_atss_loss_forward(dfm_atss_loss_t* h, const float* const* d_cls,
                          const float* const* d_bbox, const float* const* d_centerness,
                          const float* d_gt_boxes, const int* d_gt_labels, const int* d_gt_off,
                          const int* h_gt_off, const int* h_pad_shape, float* const* d_grad_cls,
                          float* const* d_grad_bbox, float* const* d_grad_centerness,
                          float* d_norm, void* stream);
/* From the last forward and d_avg [2] (d_norm, or its mean over ranks): d_losses [3][L]
 * (loss_cls, loss_bbox, loss_centerness of each level) and d_scales [3][L], the factor each
 * stored gradient takes to become that of its loss. */
int dfm_atss_loss_finish(dfm_atss_loss_t* h, const float* d_avg, float* d_losses,
                         float* d_scales, void* stream);
/* Test hook, from the last forward, [batch][N] per anchor (N over all levels): "assigned_gt"
 * int32 (0 negative or invalid, g + 1 for the image's GT g), "labels" int32 (C for negatives
 * and invalid anchors), "label_weights" fp32, "centerness_targets" fp32 (0 for non-positives),
 * "bbox_targets" fp32 [batch][N][4]; "thresholds" fp32 [G], each GT's IoU threshold.
 * DFM_ERR_STATE before a forward, DFM_ERR_INVALID on an unknown name or wrong element count. */
int dfm_atss_loss_debug_tensor(dfm_atss_loss_t* h, const char* name, void* d_out,
                               long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * DfM's LiDAR imitation loss (detectors/dfm.py:455-539 with imitation_utils.py's
 * NormalizeLayer('cw_scale') and WeightedL2WithSigmaLoss, mode 'inbox', 1x1 conv, no ReLU) for
 * `batch` samples and num_pairs (stereo x, teacher t) feature pairs per call.  Pair i has
 * channels[i] channels (16, 32 or 64) and depth[i] z slices (1 for the BEV pair): both tensors
 * are [batch][C][depth][ny][nx].  A row (b, z, y, x) is positive when the BEV cell (y, x)'s
 * anchor centre (anchor_x[x], anchor_y[y], 0) lies in one of sample b's GT boxes (mmcv's
 * points_in_boxes_part test in fp32, GT z taken as 0) and any channel of t's row is non-zero
 * (NaN counts).  With N the positives' count (its mean over ranks), w = 1 / max(N, clamp) and
 * s the [C] cw_scale buffer as it was at the call's start, pair i's loss is
 *   loss_weight[i] / batch * sum_rows w * mean_c 0.5 * (W x + bias - t / s)_c^2,
 * a NaN t / s counting as a zero difference.  In training mode, when the positives summed over
 * ranks n exceed 10, finish updates s in place: s = s * 0.99 + (sum_rows |t| / n) * 0.01 in
 * fp32.  Sums run in fp64 in a fixed order without atomics, so repeated calls are bitwise equal;
 * nothing synchronises with the host.  Create fails with DFM_ERR_INVALID on a batch outside
 * 1..64, num_pairs outside 1..2 or other channel counts.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_imitation_loss dfm_imitation_loss_t;
typedef struct dfm_imitation_loss_desc {
  int batch;                    /* B                                                          */
  int ny, nx;                   /* BEV grid                                                   */
  int num_pairs;                /* 1 or 2                                                     */
  int channels[2];              /* C of each pair                                             */
  int depth[2];                 /* z slices of each pair (1 for a BEV feature)                */
  float loss_weight[2];         /* imitation_cfg['loss_weight'] of each pair                  */
  float normalizer_clamp_value; /* the normaliser's lower clamp (10 in the shipped configs)    */
} dfm_imitation_loss_desc_t;
int dfm_imitation_loss_create(const dfm_imitation_loss_desc_t* desc, dfm_imitation_loss_t** out);
int dfm_imitation_loss_destroy(dfm_imitation_loss_t* h);
/* Device bytes the handle owns (the in-box mask and per-block partials). */
int dfm_imitation_loss_workspace(dfm_imitation_loss_t* h, long long* bytes);
/* Host arrays of num_pairs device pointers: d_stereo, d_teacher (see above), d_weight [C][C]
 * (out, in), d_bias [C], d_scale [C] (read here, updated by finish).  d_anchor_xy [nx + ny]: the
 * anchor centres' x per column, then y per row.  GT packed: d_gt_boxes [G][7] LiDAR boxes (x, y,
 * z, dx, dy, dz, yaw), d_gt_off / h_gt_off [batch + 1] on the device and the host.  Writes
 * d_packed, per pair (count / world, count, sum_rows |t_c| for each c), to be summed over ranks
 * before finish. */
int dfm_imitation_loss_forward(dfm_imitation_loss_t* h, const float* const* d_stereo,
                               const float* const* d_teacher, const float* const* d_weight,
                               const float* const* d_bias, const float* const* d_scale,
                               const float* d_anchor_xy, const float* d_gt_boxes,
                               const int* d_gt_off, const int* h_gt_off, int world,
                               float* d_packed, void* stream);
/* From the last forward and d_packed summed over ranks: d_losses [num_pairs], d_coef
 * [num_pairs] (loss_weight * w / (batch * C), the factor from pred - t to the loss's gradient)
 * and, when training, the scale update. */
int dfm_imitation_loss_finish(dfm_imitation_loss_t* h, const float* d_packed, int training,
                              float* d_losses, float* d_coef, void* stream);
/* Gradients of the last forward's losses, times d_grad_out [num_pairs] (NULL: 1), into each
 * non-null entry of the host arrays (the arrays may be NULL): d_grad_stereo (every element is
 * written, zero outside the positives), d_grad_weight [C][C] and d_grad_bias [C].  Reads the
 * workspace the last forward wrote: call it before the next forward. */
int dfm_imitation_loss_backward(dfm_imitation_loss_t* h, const float* d_coef,
                                const float* d_grad_out, float* const* d_grad_stereo,
                                float* const* d_grad_weight, float* const* d_grad_bias,
                                void* stream);
/* Test hook, from the last forward: "inbox" uint8 [batch][ny][nx], "counts" int32 [num_pairs]
 * (this rank's positives), "loss_sums" fp64 [num_pairs] (sum_rows sum_c 0.5 * diff^2).
 * DFM_ERR_STATE before a forward, DFM_ERR_INVALID on an unknown name or wrong element count. */
int dfm_imitation_loss_debug_tensor(dfm_imitation_loss_t* h, const char* name, void* d_out,
                                    long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * DepthHead.loss (dense_heads/depth_head.py:75-188) and its gradient for num_images = B * N
 * images per call, types ce / balanced_ce / focal / balanced_focal: per masked pixel
 *   w_pix * sum_k p_k * alpha * (1 - P_k)^gamma * (-log P_k),
 * log P the fp32 log-softmax over the f * D bins, p_k = 1 - min(|s_k - gt| / (s_1 - s_0), 1),
 * mask (gt > min_depth) & (gt < max_depth) in fp32 (NaN and inf excluded), w_pix fg_weight /
 * bg_weight by the foreground mask for the balanced types and 1 otherwise.  The loss is
 * loss_weight^2 * sum / (masked pixels of all images): the reference multiplies by its
 * loss_weight and by a per-type weight that equals it.  The ce types are alpha = 1, gamma = 0.
 * dense = 0: the bins are the x-factor trilinear (align_corners) upsampling of the low-res
 * logits [num_images][num_planes][height][width], read column by column (DepthHead.forward's
 * arithmetic); nothing of the size of the full-resolution volume is allocated.  dense = 1 (factor
 * 1): the input is the full-resolution volume itself.  No host synchronisation inside forward;
 * sums run in a fixed order (fp32 per pixel, fp64 across pixels), so repeated calls are bitwise
 * equal.  Create fails with DFM_ERR_INVALID on an empty shape, fewer than two bins, factor != 1
 * with dense, or num_images * num_planes > 65535.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_depth_loss dfm_depth_loss_t;
typedef struct dfm_depth_loss_desc {
  int num_images;               /* B * N                                                      */
  int num_planes, height, width;/* D, H, W of the input                                       */
  int factor;                   /* DepthHead.downsample_factor (1 with dense)                 */
  int dense;                    /* 1: the input is the full-resolution volume                 */
  float min_depth, max_depth;   /* depth_cfg                                                  */
  float alpha, gamma;           /* focal factor; 1 and 0 for the ce types                     */
  float fg_weight, bg_weight;   /* balanced types                                             */
  int balanced;
  float loss_weight;            /* depth_loss['loss_weight'], applied squared                 */
} dfm_depth_loss_desc_t;
int dfm_depth_loss_create(const dfm_depth_loss_desc_t* desc, dfm_depth_loss_t** out);
int dfm_depth_loss_destroy(dfm_depth_loss_t* h);
/* Device bytes the handle owns (per-pixel records and per-block partials). */
int dfm_depth_loss_workspace(dfm_depth_loss_t* h, long long* bytes);
/* d_volume: the logits or the dense volume; d_samples [f * D] fp32 bin depths; d_depth
 * [num_images][f * height][f * width] fp32; d_fgmask the same shape, uint8 (non-zero =
 * foreground), required by the balanced types and ignored by the others; d_empty [1] or NULL: the
 * loss returned when no pixel is masked (0 when NULL).  d_grad, when not NULL, receives the
 * gradient of the unweighted, unnormalised sum with respect to d_volume (same layout; zero
 * outside the masked columns of a dense volume).  d_loss [1] the loss, d_scale [1] the factor the
 * stored gradient takes to become the loss's (0 when no pixel is masked). */
int dfm_depth_loss_forward(dfm_depth_loss_t* h, const float* d_volume, const float* d_samples,
                           const float* d_depth, const unsigned char* d_fgmask,
                           const float* d_empty, float* d_grad, float* d_loss, float* d_scale,
                           void* stream);
/* Test hook, from the last forward: "pixel_loss" fp32 [num_images][f * height][f * width], the
 * weighted per-pixel term (0 outside the mask); "count" int32 [1], the masked pixels.
 * DFM_ERR_STATE before a forward, DFM_ERR_INVALID on an unknown name or wrong element count. */
int dfm_depth_loss_debug_tensor(dfm_depth_loss_t* h, const char* name, void* d_out,
                                long long numel, void* stream);

/* ------------------------------------------------------------------------------------
 * KITTI evaluation (mmdet3d kitti_utils/eval.py: eval_class of every requested metric) of N
 * frames of ground truth and detections in CSR form.  Per box, fp64:
 *   gt [num_gt][14]: bbox[4] alpha location[3] dimensions[3] rotation_y occluded truncated
 *   dt [num_dt][13]: bbox[4] alpha location[3] dimensions[3] rotation_y score
 * gt_code: class id (0 Car, 1 Pedestrian, 2 Cyclist, 3 Van, 4 Person_sitting, 7 other), plus 8
 * when the name is exactly "DontCare"; dt_code: class id.  gt_off / dt_off [N + 1] int32,
 * pair_off [N + 1] int64 (sum of dt * gt counts of earlier frames), num_pairs = pair_off[N].
 * A config is (metric slot, class slot, difficulty, overlap set), index
 * ((m * num_classes + c) * 3 + difficulty) * 2 + k; there are num_metrics * num_classes * 6.
 * ---------------------------------------------------------------------------------- */
typedef struct dfm_kitti_eval dfm_kitti_eval_t;
typedef struct dfm_kitti_eval_desc {
  int num_classes;               /* 1..3                                                  */
  int classes[3];                /* 0 Car, 1 Pedestrian, 2 Cyclist                         */
  int num_metrics;               /* 1..3                                                  */
  int metrics[3];                /* ascending: 0 bbox, 1 bev, 2 3d                         */
  int compute_aos;               /* AOS similarity on the bbox metric                      */
  int f32_flags;                 /* input arrays the caller held as float32: 1 gt bbox, 2 dt
                                    bbox, 4 gt 3-D box, 8 dt 3-D box, 16 gt (bbox, alpha),
                                    32 dt (bbox, alpha, score)                              */
  double min_overlap[3][3][2];   /* [metric slot][class slot][overlap set]                 */
} dfm_kitti_eval_desc_t;
int dfm_kitti_eval_create(const dfm_kitti_eval_desc_t* desc, dfm_kitti_eval_t** out);
int dfm_kitti_eval_destroy(dfm_kitti_eval_t* h);
/* The forward evaluates the frames in parts: runs of whole frames whose overlaps (num_metrics
 * fp64 per (detection, GT) pair) fit `bytes` (default 4 GiB).  The rest of the workspace is
 * O(frames + GT + detections).  The results are bitwise the same for every limit; a frame
 * whose own overlaps exceed the limit is refused with DFM_ERR_INVALID.  With more than one
 * part the forward reads pair_off back to the host and synchronises the stream. */
int dfm_kitti_eval_set_overlap_limit(dfm_kitti_eval_t* h, long long bytes);
/* The last forward's workspace in bytes, its overlap buffer in bytes, and its part count;
 * DFM_ERR_STATE before a forward. */
int dfm_kitti_eval_workspace(const dfm_kitti_eval_t* h, long long* workspace_bytes,
                             long long* overlap_bytes, int* num_parts);
/* d_pr: device [configs][41][4] fp64 (tp, fp, fn, similarity per threshold; zero past the
 * count); d_thr_count: device [configs] int32, 42 when a config has more thresholds than the
 * reference's 41-point arrays hold; d_status: device int32, 0 on success, bit 0 set when a
 * frame holds more than 1024 detections (the limit per frame; such a frame is not evaluated
 * and the counts are not valid).  The caller reads d_status after the stream completes.
 * The workspace grows on demand. */
int dfm_kitti_eval_forward(dfm_kitti_eval_t* h, int num_frames, int num_gt, int num_dt,
                           long long num_pairs, const double* d_gt, const int* d_gt_code,
                           const int* d_gt_off, const double* d_dt, const int* d_dt_code,
                           const int* d_dt_off, const long long* d_pair_off, double* d_pr,
                           int* d_thr_count, int* d_status, void* stream);
/* Test hook, from the last forward: "overlap<metric>" fp64 [pairs of the last part] ([dt][gt]
 * per frame; all num_pairs when the set fit in one part),
 * "tp_scores" fp64 [configs][S] (each config's TP scores sorted descending, S = the power of
 * two >= num_gt), "tp_count" int32 [configs], "thresholds" fp64 [configs][41],
 * "num_valid_gt" int32 [num_classes * 3].  DFM_ERR_STATE before a forward, DFM_ERR_INVALID on
 * an unknown name or a wrong element count. */
int dfm_kitti_eval_debug_tensor(dfm_kitti_eval_t* h, const char* name, void* d_out,
                                long long numel, void* stream);
/* rotate_iou_gpu_eval: d_iou [n][k] = IoU of (d_qboxes[k], d_boxes[n]) by criterion (-1 IoU,
 * 0 / 1 over the first / second box's area, 2 intersection area); boxes [.][5] fp32
 * (x, z, l, w, ry) in camera BEV. */
int dfm_op_eval_rotated_iou(const float* d_boxes, const float* d_qboxes, int n, int k,
                            int criterion, float* d_iou, void* stream);

/* ------------------------------------------------------------------------------------
 * Pair stage of Waymo's camera-only LET-3D-AP (compute_detection_let_metrics_main).
 * d_pred [n][7], d_gt [k][7]: fp64 boxes (center x, y, z, length, width, height, heading)
 * in the vehicle frame.  d_out [n][k][3] fp64: for prediction i and GT j, the 3-D rotated
 * IoU of the prediction aligned along the sensor -> prediction ray to the point closest to
 * the GT centre (LET-IoU), the longitudinal affinity 1 - min(|e_lon| / tol, 1) with
 * tol = max(0.1 |c_gt - s|, 0.5 m) and s = (1.43, 0, 2.18), and the heading accuracy
 * 1 - |wrapped heading error| / pi.
 * ---------------------------------------------------------------------------------- */
int dfm_op_let_iou(const double* d_pred, const double* d_gt, int n, int k, double* d_out,
                   void* stream);

/* ------------------------------------------------------------------------------------
 * WaymoDataset.convert_valid_bboxes + bbox2result_kitti (mmdet3d datasets/waymo_dataset.py)
 * for load_mode 'lidar_frame', for a whole set in one launch.  d_boxes [num_boxes][7] fp32
 * LiDAR boxes (x, y, z, dx, dy, dz, yaw; bottom centre), d_box_off [num_frames + 1] int32;
 * per frame d_calib [num_frames][32] fp32 (R0_rect @ Tr_velo_to_cam as float32 [4][4], then
 * P0 [4][4]), d_image_shape [num_frames][2] int32 (H, W), d_image_idx [num_frames] int64;
 * limit_range: host float[6] (x0, y0, z0, x1, y1, z1).  Writes per box d_keep (1 iff the
 * centre lies strictly inside limit_range), d_sample_idx (its frame's image_idx) and d_out
 * [num_boxes][17] fp32: the 2-D box from the P0 projection of the camera box's corners,
 * clipped to the image (x0, y0, x1, y1), alpha, camera location[3], dimensions[3] (l, h, w),
 * rotation_y, the LiDAR yaw after limit_yaw(0.5, 2 pi), and the 2-D box before clipping. */
int dfm_waymo_kitti_convert(int num_frames, int num_boxes, const float* d_boxes,
                            const int* d_box_off, const float* d_calib, const int* d_image_shape,
                            const long long* d_image_idx, const float* limit_range,
                            unsigned char* d_keep, float* d_out, long long* d_sample_idx,
                            void* stream);

/* ------------------------------------------------------------------------------------
 * Image preparation of the shipped test pipelines, one launch per batch of views.
 * d_src: num_views decoded 8-bit BGR images, [num_views][src_h][src_w][3], all one size.
 * d_out: [num_views][3][pad_h][pad_w] fp32, pad_h / pad_w = out_h / out_w rounded up to
 * pad_divisor; every element is written (pad cells 0).
 *   DFM_IMAGE_PREP_CROP    (KITTI): the window img[crop_y:crop_y+out_h, crop_x:crop_x+out_w]
 *                          (RandomCrop3D), which must lie inside the image.
 *   DFM_IMAGE_PREP_RESCALE (Waymo): cv2.resize(INTER_LINEAR) of the float image to
 *                          out_w x out_h (mmcv.imrescale); an exact 2x downscale, which cv2
 *                          runs as INTER_AREA, is refused.
 * Then mmcv.imnormalize (as cv2 computes it): channel swap if to_rgb, then
 * float(double(x - float(mean[c])) * (1 / std[c])), and
 * impad_to_multiple(pad_divisor, pad_val=0).  DFM_ERR_INVALID for sizes it cannot serve.
 * ---------------------------------------------------------------------------------- */
#define DFM_IMAGE_PREP_CROP 0
#define DFM_IMAGE_PREP_RESCALE 1
typedef struct dfm_image_prep_desc {
  int mode;            /* DFM_IMAGE_PREP_CROP or DFM_IMAGE_PREP_RESCALE            */
  int num_views;       /* views stacked in d_src and d_out                         */
  int src_h, src_w;    /* decoded view size                                        */
  int crop_x, crop_y;  /* crop: window origin (ignored by rescale)                 */
  int out_h, out_w;    /* crop: window size; rescale: resized size                 */
  int pad_divisor;     /* Pad / MultiViewImagePad size_divisor                      */
  int to_rgb;          /* 1: BGR -> RGB before normalising                         */
  double mean[3];      /* img_norm_cfg mean, per output channel, as stored by the     */
  double std[3];       /* Normalize transforms: fp32 values (widened), not the config's */
} dfm_image_prep_desc_t;
int dfm_image_prep(const dfm_image_prep_desc_t* desc, const unsigned char* d_src, float* d_out,
                   void* stream);

/* Re-entrancy: handles may live on different devices and be driven from different host
 * threads only if each thread owns its device; per-device scratch (K-slice partial sums,
 * lifting staging, the host-copy side stream) and the profiling record are shared by all
 * handles of a device and are NOT locked -- the same one-thread-per-process model as the
 * reference (tools/slurm_train.sh:15-24, SURVEY.md section 8b "Threading"). */

/* ------------------------------------------------------------------------------------
 * The per-view image-feature cache of the detectors (modules.DfM.set_feature_cache).
 *
 * dfm_view_fingerprint: a 128-bit fingerprint of each of num_views consecutive views of
 * view_elems fp32 elements (d_views 4-byte aligned), in one launch.  d_out[v][0..1] are two
 * 64-bit lanes: lane j is the sum modulo 2^64 over elements i of y ^ (y >> 32), y =
 * (((bits(x_i) << 32) ^ i ^ K_j) * M_j) mod 2^64 (view_cache_kernels.cuh).  The raw bits are hashed, so
 * -0.0 != +0.0 and NaN payloads count; the result does not depend on thread order.
 * ---------------------------------------------------------------------------------- */
int dfm_view_fingerprint(const float* d_views, int num_views, long long view_elems,
                         unsigned long long* d_out /* [num_views][2] */, void* stream);
/* Compares num_pairs view pairs of view_elems fp32 elements bit for bit (h_a / h_b: host
 * arrays of device pointers).  d_mismatch[i] = 1 when pair i differs in any bit, else 0.  One
 * launch per 64 pairs. */
int dfm_views_equal(const float* const* h_a, const float* const* h_b, int num_pairs,
                    long long view_elems, int* d_mismatch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFM_B200_H_ */
