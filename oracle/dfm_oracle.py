"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference DfM hot path.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline``
/ ``--impl reference`` legs may import this module, and only as the checker or
as the timed CPU baseline.  The product (``depth_from_motion_b200``) never
imports it and has no CPU fallback.

What this is
------------
A function-by-function restatement, in plain fp32 PyTorch-CPU calls, of the path
SURVEY.md section 8(a) lists, each function citing the reference file:line it
follows (paths relative to the reference checkout, commit e2321189):

    a1  build_dfm_cost      mmdet3d/models/backbones/dfm_backbone.py:217-314
    a2  DfMBackbone.forward mmdet3d/models/backbones/dfm_backbone.py:143-214
    a3  hourglass           mmdet3d/models/utils/conv_modules.py:73-149
    a4  pred + gate         mmdet3d/models/backbones/dfm_backbone.py:118-141
    a5  DepthHead.forward   mmdet3d/models/dense_heads/depth_head.py:190-212
    a6  point_sample + MultiViewDfM.feature_transformation
                            mmdet3d/models/fusion_layers/point_fusion.py:14-106
                            mmdet3d/models/detectors/multiview_dfm.py:119-209
    a7  DfMNeck / OutdoorImVoxelNeck / ResModule
                            mmdet3d/models/necks/dfm_neck.py:10-122
                            mmdet3d/models/necks/imvoxel_neck.py:8-117
    a8  voxel_sample        mmdet3d/models/fusion_layers/point_fusion.py:324-410
                            (oracle only: no shipped config reaches it, SURVEY.md 8a)
    a9  points_cam2img / points_img2cam
                            mmdet3d/core/bbox/structures/utils.py:176-248
    f1  FrustumToVoxel.forward (SURVEY.md section 8(f) row 1)
                            mmdet3d/models/necks/feature_transformation.py:68-187
                            mmdet3d/models/detectors/dfm.py:174-211 (voxel grid)
    f2  SPPUNetNeck.lastconv (section 8(f) row 2)
                            mmdet3d/models/necks/spp_unet_neck.py:60-75, :110
    f3  BEVHourglass.forward + LIGAAnchor3DHead.forward_single (section 8(f) row 3)
                            mmdet3d/models/backbones/bev_hourglass.py:11-137
                            mmdet3d/models/dense_heads/liga_anchor3d_head.py:37-128
                            mmdet3d/models/detectors/dfm.py:426-432

Third-party arithmetic: every number on this path is produced by PyTorch ATen
ops in the reference (README pins torch 1.9 + mmcv-full 1.6.0, the latter used
for ConvModule *wiring* only).  The restatement therefore calls the same ATen
ops on CPU (conv3d, conv_transpose3d, group_norm(eps=1e-5), batch_norm,
grid_sample, interpolate(trilinear), softmax, inverse) in the same order with
the same argument values; parameters are passed as a flat dict keyed by the
reference ``state_dict`` names.

Pinning (SURVEY.md section 8c)
------------------------------
The reference's own tests hold golden vectors only for the geometry helpers
(tests/test_utils/test_utils.py:186-193, tests/test_utils/test_box3d.py:1653-1680)
and ``point_sample`` (tests/test_models/test_fusion/test_point_fusion.py:13-58);
those are reproduced in tests/test_oracle_golden.py.  For build_dfm_cost /
DfMBackbone / DepthHead / DfMNeck / FrustumToVoxel the reference has NO tests, so this
restatement is pinned against outputs of the reference's own source files
executed verbatim in the build container (oracle/ref_loader.py), committed as
fixtures under tests/golden/ by tests/golden/make_golden.py.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

GN_EPS = 1e-5  # nn.GroupNorm default, conv_modules.py:42-43


# ----------------------------------------------------------------------------
# a9  geometry helpers
# ----------------------------------------------------------------------------
def points_cam2img(points_3d, proj_mat, with_depth=False):
    """core/bbox/structures/utils.py:176-214."""
    d1, d2 = proj_mat.shape[:2]
    assert (d1, d2) in ((3, 3), (3, 4), (4, 4))
    if d1 == 3:
        expanded = torch.eye(4, dtype=proj_mat.dtype, device=proj_mat.device)
        expanded[:d1, :d2] = proj_mat
        proj_mat = expanded
    ones = points_3d.new_ones(list(points_3d.shape[:-1]) + [1])
    points_4 = torch.cat([points_3d, ones], dim=-1)
    point_2d = points_4 @ proj_mat.T
    res = point_2d[..., :2] / point_2d[..., 2:3]
    if with_depth:
        res = torch.cat([res, point_2d[..., 2:3]], dim=-1)
    return res


def points_img2cam(points, cam2img):
    """core/bbox/structures/utils.py:217-248."""
    assert cam2img.shape[0] <= 4 and cam2img.shape[1] <= 4
    assert points.shape[1] == 3
    xys = points[:, :2]
    depths = points[:, 2].view(-1, 1)
    unnormed_xys = torch.cat([xys * depths, depths], dim=1)
    pad = torch.eye(4, dtype=xys.dtype, device=xys.device)
    pad[:cam2img.shape[0], :cam2img.shape[1]] = cam2img
    inv_pad = torch.inverse(pad).transpose(0, 1)
    n = unnormed_xys.shape[0]
    homo = torch.cat([unnormed_xys, xys.new_ones((n, 1))], dim=1)
    return torch.mm(homo, inv_pad)[:, :3]


# ----------------------------------------------------------------------------
# a1  plane-sweep volume
# ----------------------------------------------------------------------------
def build_dfm_cost(cur_feats, prev_feats, depths, feat_sample_factor,
                   cost_sample_factor, cam2imgs, cur2prevs, img_shape,
                   flip=False, img_crop_offset=(0, 0), img_scale_factor=1.0):
    """dfm_backbone.py:217-314.  Returns [B, 2C, D, Ho, Wo]."""
    dev = cur_feats.device  # the reference builds everything on the feature's device (:238)
    crop = torch.tensor(img_crop_offset, device=dev)
    depths = depths.to(dev)
    batch_size = cur_feats.shape[0]
    h_in, w_in = cur_feats.shape[-2:]
    num_depths = depths.shape[-1]
    h_out = round(h_in / cost_sample_factor)
    w_out = round(w_in / cost_sample_factor)
    ws = torch.linspace(0, w_out - 1, w_out, device=dev) * feat_sample_factor * \
        cost_sample_factor                                        # :247-248
    hs = torch.linspace(0, h_out - 1, h_out, device=dev) * feat_sample_factor * \
        cost_sample_factor                                        # :249-250
    ds_3d, ys_3d, xs_3d = torch.meshgrid(depths, hs, ws, indexing='ij')
    grid = torch.stack([xs_3d, ys_3d, ds_3d], dim=-1)            # :253
    grid = grid[None].repeat(batch_size, 1, 1, 1, 1)
    for idx in range(batch_size):                                 # :257-271
        grid[..., :2] += crop
        grid[..., :2] /= img_scale_factor
        if flip:
            org_h, org_w = img_shape
            grid[..., 0] = org_w - grid[..., 0]
        grid3d = points_img2cam(grid[idx].view(-1, 3), cam2imgs[idx][:3])
        pad_ones = grid3d.new_ones(grid3d.shape[0], 1)
        homo_grid3d = torch.cat([grid3d, pad_ones], dim=1)
        cur_grid = points_cam2img(grid3d, cam2imgs[idx])[:, :2]
        prev_grid3d = (homo_grid3d @ cur2prevs[idx].transpose(0, 1))[:, :3]
        prev_grid = points_cam2img(prev_grid3d, cam2imgs[idx])[:, :2]
    cur_grid = cur_grid.view(batch_size, 1, -1, 2)
    prev_grid = prev_grid.view(batch_size, 1, -1, 2)
    if flip:                                                      # :278-281
        org_h, org_w = img_shape
        cur_grid[..., 0] = org_w - cur_grid[..., 0]
        prev_grid[..., 0] = org_w - prev_grid[..., 0]
    cur_grid *= img_scale_factor
    prev_grid *= img_scale_factor
    cur_grid -= crop
    prev_grid -= crop
    cur_grid /= feat_sample_factor
    prev_grid /= feat_sample_factor
    cur_grid[..., 0] = cur_grid[..., 0] / (w_in - 1) * 2 - 1     # :291-294
    cur_grid[..., 1] = cur_grid[..., 1] / (h_in - 1) * 2 - 1
    prev_grid[..., 0] = prev_grid[..., 0] / (w_in - 1) * 2 - 1
    prev_grid[..., 1] = prev_grid[..., 1] / (h_in - 1) * 2 - 1
    # the grid keeps the reference's fp32 geometry; fp64 features sample it exactly widened
    cur_cost = F.grid_sample(cur_feats, cur_grid.to(cur_feats.dtype), mode='bilinear',
                             padding_mode='zeros', align_corners=True)
    cur_cost = cur_cost.view(batch_size, -1, num_depths, h_out, w_out)
    prev_cost = F.grid_sample(prev_feats, prev_grid.to(prev_feats.dtype), mode='bilinear',
                              padding_mode='zeros', align_corners=True)
    prev_cost = prev_cost.view(batch_size, -1, num_depths, h_out, w_out)
    return torch.cat([cur_cost, prev_cost], dim=1)                # :313


# ----------------------------------------------------------------------------
# a2-a4  3-D aggregation.  `q` is an optional operand-rounding hook used only by
# the precision study in DESIGN.md (identity by default => exact restatement).
# ----------------------------------------------------------------------------
def _ident(x):
    return x


def _q(q, t, layer, kind):
    """Operand-rounding hook of the precision study (tools/precision_study.py): `q` is either
    a one-argument function applied to every conv operand, or an object with a
    ``round(tensor, layer, kind)`` method (kind 'x' = activation, 'w' = weight) that can treat
    each of the 22 conv layers differently.  Identity by default."""
    r = getattr(q, 'round', None)
    return r(t, layer, kind) if r is not None else q(t)


def _gn(x, p, prefix, groups=32):
    return F.group_norm(x, groups, p[prefix + '.weight'], p[prefix + '.bias'],
                        GN_EPS)


def _conv_module(x, p, name, act=True, q=_ident):
    """mmcv ConvModule(conv3d k3 s1 p1, bias=False) -> GN(32) -> [ReLU];
    dfm_backbone.py:50-66, 118-127."""
    y = F.conv3d(_q(q, x, name, 'x'), _q(q, p[name + '.conv.weight'], name, 'w'), None, 1, 1)
    y = _gn(y, p, name + '.gn')
    return F.relu(y) if act else y


def hourglass(x, p, name, q=_ident):
    """conv_modules.py:129-149 with presqu = postsqu = None (dfm_backbone.py:181)."""
    def cb(t, sub, stride):  # convbn_3d, conv_modules.py:27-43
        ln = f'{name}.{sub}'
        y = F.conv3d(_q(q, t, ln, 'x'), _q(q, p[f'{name}.{sub}.0.weight'], ln, 'w'), None,
                     stride, 1)
        return _gn(y, p, f'{name}.{sub}.1')

    def cb_seq(t, sub, stride):  # nn.Sequential(convbn_3d, ReLU)
        ln = f'{name}.{sub}'
        y = F.conv3d(_q(q, t, ln, 'x'), _q(q, p[f'{name}.{sub}.0.0.weight'], ln, 'w'), None,
                     stride, 1)
        return F.relu(_gn(y, p, f'{name}.{sub}.0.1'))

    def deconv(t, sub):  # ConvTranspose3d k3 p1 op1 s2 + GN, conv_modules.py:104-127
        ln = f'{name}.{sub}'
        y = F.conv_transpose3d(_q(q, t, ln, 'x'), _q(q, p[f'{name}.{sub}.0.weight'], ln, 'w'),
                               None, 2, 1, 1)
        return _gn(y, p, f'{name}.{sub}.1')

    out = cb_seq(x, 'conv1', 2)              # :131
    pre = F.relu(cb(out, 'conv2', 1))        # :132-136
    out = cb_seq(pre, 'conv3', 2)            # :138
    out = cb_seq(out, 'conv4', 1)            # :139
    post = F.relu(deconv(out, 'conv5') + pre)  # :145
    out = deconv(post, 'conv6')              # :147
    return out, pre, post


def _tower(x, p, sfx, q=_ident):
    """dfm_backbone.py:175-183 (stereo) / :189-197 (mono) with num_hg == 1."""
    cost0 = _conv_module(x, p, 'dres0' + sfx, True, q)
    cost0 = _conv_module(cost0, p, 'dres1' + sfx, False, q) + cost0
    hg_name = ('hg_mono' if sfx else 'hg_stereo') + '.0'
    res, _, _ = hourglass(cost0, p, hg_name, q)
    return cost0 + res


def _pred(x, p, name, q=_ident):
    """build_depth_pred_module, dfm_backbone.py:118-128."""
    y = _conv_module(x, p, name + '.0', True, q)
    return F.conv3d(_q(q, y, name + '.1', 'x'), _q(q, p[name + '.1.weight'], name + '.1', 'w'),
                    None, 1, 1)


def mono_stereo_aggregate(stereo_cost, mono_cost, p, q=_ident):
    """dfm_backbone.py:130-141."""
    cost1 = _pred(stereo_cost, p, 'pred_stereo.0', q)
    mono_cost1 = _pred(mono_cost, p, 'pred_mono.0', q)
    cost = torch.cat((cost1, mono_cost1), dim=1).flatten(1, 2)
    weight = F.conv2d(cost, p['aggregate_cost.weight']).unsqueeze(1).sigmoid()
    return weight * cost1 + (1 - weight) * mono_cost1


def aggregate_volume(cost_raw, p, in_channels=32, q=_ident):
    """DfMBackbone.forward after build_dfm_cost, dfm_backbone.py:174-214."""
    cur_cost = _tower(cost_raw, p, '', q)
    cur_cost_mono = _tower(cost_raw[:, :in_channels], p, '_mono', q)
    cost = mono_stereo_aggregate(cur_cost, cur_cost_mono, p, q)
    return cost, cur_cost, cur_cost_mono


def downsampled_depth(depth_cfg):
    """DfM.prepare_depth, detectors/dfm.py:147-168 (plane centres, offset 0.5)."""
    nb, ds = depth_cfg['num_bins'], depth_cfg['downsample_factor']
    interval = (depth_cfg['depth_max'] - depth_cfg['depth_min']) / nb
    d = torch.zeros(nb // ds, dtype=torch.float32)
    for i in range(nb // ds):
        d[i] = (i + 0.5) * ds * interval + depth_cfg['depth_min']
    return d


def depth_samples(depth_cfg):
    """DfM.prepare_depth, detectors/dfm.py:169-172 (full-resolution bin centres)."""
    nb = depth_cfg['num_bins']
    interval = (depth_cfg['depth_max'] - depth_cfg['depth_min']) / nb
    d = torch.zeros(nb, dtype=torch.float32)
    for i in range(nb):
        d[i] = (i + 0.5) * interval + depth_cfg['depth_min']
    return d


def dfm_backbone_forward(p, cur_feats, prev_feats, img_metas, depth_cfg,
                         in_channels=32, cost_sample_factor=4,
                         feat_sample_factor=1, q=_ident):
    """DfMBackbone.forward, dfm_backbone.py:143-214."""
    dev = cur_feats.device
    ori_cam2imgs = torch.as_tensor(
        np.array([m['ori_cam2img'] for m in img_metas]), dtype=torch.float32).to(dev)
    cur2prevs = torch.stack([torch.as_tensor(np.asarray(m['cur2prevs']),
                                             dtype=torch.float32)
                             for m in img_metas]).to(dev)
    cost_raw = build_dfm_cost(
        cur_feats, prev_feats, downsampled_depth(depth_cfg),
        feat_sample_factor, cost_sample_factor, ori_cam2imgs, cur2prevs[0],
        img_metas[0]['ori_shape'][:2], img_metas[0].get('flip', False),
        img_metas[0]['crop_offset'],
        img_scale_factor=img_metas[0].get('scale_factor', [1.0])[0])
    return aggregate_volume(cost_raw, p, in_channels, q)


# ----------------------------------------------------------------------------
# a5  DepthHead.forward (with_convs=False, the KITTI config)
# ----------------------------------------------------------------------------
def depth_head_forward(cost, samples, downsample_factor=4):
    """depth_head.py:190-212: x4 trilinear (align_corners) -> softmax(D) ->
    expectation over the full-resolution bin centres."""
    vol = F.interpolate(cost, scale_factor=downsample_factor, mode='trilinear',
                        align_corners=True)
    sm = F.softmax(vol, dim=2)
    preds = torch.sum(sm * samples.to(vol.device)[None, None, :, None, None], 2)
    return vol, sm, preds


# ----------------------------------------------------------------------------
# a6  multi-view voxel lifting
# ----------------------------------------------------------------------------
def point_sample(img_features, points, proj_mat, img_scale_factor,
                 img_crop_offset, img_flip, img_pad_shape, img_shape,
                 aligned=True, valid_flag=False):
    """point_fusion.py:14-106 with apply_3d_transformation == identity (no 3-D
    augmentation keys in img_meta at test time, coord_transform.py:9-92)."""
    if valid_flag:
        proj = points_cam2img(points, proj_mat, with_depth=True)
        pts_2d, depths = proj[..., :2], proj[..., 2]
    else:
        pts_2d = points_cam2img(points, proj_mat)
    img_coors = pts_2d[:, 0:2] * img_scale_factor
    img_coors = img_coors - img_crop_offset
    coor_x, coor_y = torch.split(img_coors, 1, dim=1)
    if img_flip:
        ori_h, ori_w = img_shape
        coor_x = ori_w - coor_x
    h, w = img_pad_shape
    norm_y = coor_y / h * 2 - 1
    norm_x = coor_x / w * 2 - 1
    grid = torch.cat([norm_x, norm_y], dim=1).unsqueeze(0).unsqueeze(0)
    mode = 'bilinear' if aligned else 'nearest'
    if aligned or img_features.dtype == grid.dtype:
        feats = F.grid_sample(img_features, grid.to(img_features.dtype), mode=mode,
                              padding_mode='zeros', align_corners=True)
    else:
        # wider features (fp64 reference runs): the tap is the one grid_sample picks in the
        # geometry's precision, found by sampling a map of 1-based pixel indices, and its value
        # is gathered exactly
        hf, wf = img_features.shape[-2:]
        tags = torch.arange(1, hf * wf + 1, dtype=grid.dtype, device=grid.device)
        tap = F.grid_sample(tags.view(1, 1, hf, wf), grid, mode='nearest',
                            padding_mode='zeros', align_corners=True).view(-1).long()
        flat = img_features.reshape(img_features.shape[1], hf * wf)
        feats = (flat[:, (tap - 1).clamp(min=0)] * (tap > 0))[None, :, None]
    if valid_flag:
        valid = (coor_x.squeeze() < w) & (coor_x.squeeze() > 0) & \
            (coor_y.squeeze() < h) & (coor_y.squeeze() > 0) & (depths > 0)
        vf = feats.squeeze().t().clone()
        vf[~valid] = 0
        return vf, valid
    return feats.squeeze().t()


def voxel_centers(n_voxels, point_cloud_range):
    """AlignedAnchor3DRangeGenerator.grid_anchors -> [:, :3]
    (core/anchor/anchor_3d_generator.py:225-341 as configured at
    detectors/multiview_dfm.py:54-61,122-123): centres ordered z-major,
    then y, then x fastest ... reshaped by the caller as [Nz, Ny, Nx]."""
    nx, ny, nz = n_voxels
    x0, y0, z0, x1, y1, z1 = point_cloud_range
    vx, vy, vz = (x1 - x0) / nx, (y1 - y0) / ny, (z1 - z0) / nz
    xs = torch.arange(nx, dtype=torch.float32) * vx + (x0 + vx / 2)
    ys = torch.arange(ny, dtype=torch.float32) * vy + (y0 + vy / 2)
    zs = torch.arange(nz, dtype=torch.float32) * vz + (z0 + vz / 2)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    return torch.stack([xx, yy, zz], dim=-1).reshape(-1, 3)


def multiview_lift(feats, points, n_voxels, lidar2imgs, num_views, num_frames,
                   img_scale_factor, img_crop_offset, img_flip, input_shape,
                   img_shapes, temporal_aggregate='mean'):
    """MultiViewDfM.feature_transformation, multiview_dfm.py:139-209, one sample,
    valid_sample=True.  feats [T*Nv, C, H, W] -> [C(*T), Nx, Ny, Nz]."""
    frame_volume, frame_valid = [], []
    for f in range(num_frames):
        vol, flags = [], []
        for v in range(num_views):
            s = f * num_views + v
            vf, valid = point_sample(
                feats[s][None], points, lidar2imgs[s], img_scale_factor,
                img_crop_offset, img_flip, input_shape, img_shapes[s][:2],
                aligned=False, valid_flag=True)
            vol.append(vf)
            flags.append(valid)
        nums = torch.stack(flags, 0).sum(0)
        volume = torch.stack(vol, 0).sum(0)
        volume[~(nums > 0)] = 0
        frame_volume.append(volume)
        frame_valid.append(nums)
    if temporal_aggregate == 'mean':
        fv = torch.stack(frame_volume, 0).sum(0)
        fn = torch.stack(frame_valid, 0).sum(0)
        fv[~(fn > 0)] = 0
        fv = fv / torch.clamp(fn[:, None], min=1)
    else:  # 'concat'
        fn = torch.stack(frame_valid, 1)
        fv = torch.stack(frame_volume, 1)
        fv[~(fn > 0)] = 0
        fv = (fv / torch.clamp(fn[:, :, None], min=1)).flatten(1, 2)
    return fv.reshape(list(n_voxels[::-1]) + [-1]).permute(3, 2, 1, 0)


# ----------------------------------------------------------------------------
# a7  BEV necks (eval mode: BatchNorm3d uses running statistics)
# ----------------------------------------------------------------------------
def _bn(x, p, prefix):
    return F.batch_norm(x, p[prefix + '.running_mean'],
                        p[prefix + '.running_var'], p[prefix + '.weight'],
                        p[prefix + '.bias'], False, 0.0, 1e-5)


def _res_module(x, p, name):
    """imvoxel_neck.py:71-117: relu(x + BN(conv(relu(BN(conv x)))))."""
    y = F.relu(_bn(F.conv3d(x, p[name + '.conv0.conv.weight'], None, 1, 1), p,
                   name + '.conv0.bn'))
    y = _bn(F.conv3d(y, p[name + '.conv1.conv.weight'], None, 1, 1), p,
            name + '.conv1.bn')
    return F.relu(x + y)


def _neck_tower(x, p, name):
    """imvoxel_neck.py:27-56 / dfm_neck.py:29-88 (one tower of six layers)."""
    x = _res_module(x, p, f'{name}.0')
    x = F.relu(_bn(F.conv3d(x, p[f'{name}.1.conv.weight'], None, (1, 1, 2), 1),
                   p, f'{name}.1.bn'))
    x = _res_module(x, p, f'{name}.2')
    x = F.relu(_bn(F.conv3d(x, p[f'{name}.3.conv.weight'], None, (1, 1, 2), 1),
                   p, f'{name}.3.bn'))
    x = _res_module(x, p, f'{name}.4')
    x = F.relu(_bn(F.conv3d(x, p[f'{name}.5.conv.weight'], None, 1, (1, 1, 0)),
                   p, f'{name}.5.bn'))
    return x


def imvoxel_neck_forward(p, x):
    """OutdoorImVoxelNeck.forward, imvoxel_neck.py:58-68."""
    x = _neck_tower(x, p, 'model')
    assert x.shape[-1] == 1
    return [x[..., 0].transpose(-1, -2)]


def dfm_neck_forward(p, x, mono_channels):
    """DfMNeck.forward, dfm_neck.py:97-118."""
    mono = _neck_tower(x[:, :mono_channels], p, 'mono_layers')
    stereo = _neck_tower(x, p, 'stereo_layers')
    assert mono.shape[-1] == 1 and stereo.shape[-1] == 1
    mono = mono[..., 0].transpose(-1, -2)
    stereo = stereo[..., 0].transpose(-1, -2)
    w = F.conv2d(torch.cat([mono, stereo], 1),
                 p['aggregate_layer.weight']).sigmoid()      # :114-116
    return [w * mono + (1 - w) * stereo]                    # :117


# ----------------------------------------------------------------------------
# helpers shared by tests / bench (deterministic synthetic inputs, NumPy legacy
# MT19937 so both sides of a fixture regenerate identical tensors)
# ----------------------------------------------------------------------------
# ----------------------------------------------------------------------------
# a8  voxel_sample (frustum-from-voxel resampling; not reached by a shipped config)
# ----------------------------------------------------------------------------
def voxel_sample(voxel_features, voxel_range, voxel_size, depth_samples, proj_mat,
                 downsample_factor, img_scale_factor, img_crop_offset, img_flip,
                 img_pad_shape, img_shape, aligned=True, padding_mode='zeros',
                 align_corners=True):
    """point_fusion.py:324-410: a (depth, v, u) frustum lattice at 1/downsample_factor
    of the padded image is taken back through flip / crop / scale, unprojected with
    points_img2cam, expressed in voxel-index units (-0.5: cell centres), normalised and
    used to grid_sample the [1, C, Nx, Ny, Nz] voxel features -> [1, C, D, H, W]."""
    h, w = img_pad_shape
    h_out, w_out = round(h / downsample_factor), round(w / downsample_factor)
    ws = torch.linspace(0, w_out - 1, w_out) * downsample_factor
    hs = torch.linspace(0, h_out - 1, h_out) * downsample_factor
    depths = depth_samples[::downsample_factor]
    ds3, ys3, xs3 = torch.meshgrid(depths, hs, ws, indexing='ij')
    grid = torch.stack([xs3, ys3, ds3], dim=-1).view(-1, 3)
    if img_flip:
        grid[:, 0] = img_shape[1] - grid[:, 0]
    grid[:, :2] += img_crop_offset
    grid[:, :2] /= img_scale_factor
    grid3d = points_img2cam(grid, proj_mat)
    vr = torch.tensor(voxel_range).view(1, 6)
    vs = torch.tensor(voxel_size).view(1, 3)
    grid3d = (grid3d - vr[:, :3]) / vs - 0.5
    grid3d = grid3d / ((vr[:, 3:] - vr[:, :3]) / vs) * 2 - 1
    grid3d = grid3d.view(1, len(depths), h_out, w_out, 3)[..., [2, 1, 0]]
    return F.grid_sample(voxel_features, grid3d, mode='bilinear' if aligned else 'nearest',
                         padding_mode=padding_mode, align_corners=align_corners)


# ----------------------------------------------------------------------------
# f1  FrustumToVoxel
# ----------------------------------------------------------------------------
def frustum_coordinates_3d(voxel_cfg):
    """DfM.prepare_coordinates_3d (detectors/dfm.py:174-211, sample_rate (1,1,1)):
    pseudo-lidar voxel centres [Nz, Ny, Nx, 3] holding (x, y, z)."""
    pcr = voxel_cfg['point_cloud_range']
    vs = voxel_cfg['voxel_size']
    grid = (np.array(pcr[3:6], dtype=np.float32) -
            np.array(pcr[0:3], dtype=np.float32)) / np.array(vs)
    gx, gy, gz = np.round(grid).astype(np.int64).tolist()
    zs = torch.linspace(pcr[2] + vs[2] / 2., pcr[5] - vs[2] / 2., gz,
                        dtype=torch.float32)
    ys = torch.linspace(pcr[1] + vs[1] / 2., pcr[4] - vs[1] / 2., gy,
                        dtype=torch.float32)
    xs = torch.linspace(pcr[0] + vs[0] / 2., pcr[3] - vs[0] / 2., gx,
                        dtype=torch.float32)
    zs, ys, xs = torch.meshgrid(zs, ys, xs, indexing='ij')
    return torch.stack([xs, ys, zs], dim=-1).float()


def frustum_grid(coordinates_3d, cam2img, pad_shape, depth_cfg):
    """feature_transformation.py:84-124 for one sample: pseudo-lidar -> rect
    camera (x,y,z) -> (-y,-z,x) (:175-177), pixel = P[:3] [X,Y,Z,1] / w
    (:180-187), third coordinate = rect depth; normalisation by the padded image
    size and the depth range; the two validity masks."""
    c3d = coordinates_3d.reshape(-1, 3)
    rect = torch.stack([-c3d[:, 1], -c3d[:, 2], c3d[:, 0]], dim=-1)
    P = torch.as_tensor(cam2img, dtype=torch.float32)[:3].float()
    hom = torch.cat([rect, torch.ones((rect.shape[0], 1))], dim=1)
    pts = torch.mm(hom, P.t())
    pts[:, 0] /= pts[:, 2]
    pts[:, 1] /= pts[:, 2]
    coord = torch.cat([pts[:, 0:2], rect[:, 2:]], dim=-1)
    coord = coord.view(*coordinates_3d.shape[:3], 3)
    valid2d = ((coord[..., 0] >= 0) & (coord[..., 0] <= pad_shape[1]) &
               (coord[..., 1] >= 0) & (coord[..., 1] <= pad_shape[0]))
    lo = torch.as_tensor([0, 0, depth_cfg['depth_min']])
    span = torch.as_tensor([pad_shape[1] - 1, pad_shape[0] - 1,
                            depth_cfg['depth_max'] - depth_cfg['depth_min']])
    norm = (coord - lo) / span
    norm = norm * 2. - 1.
    valid = valid2d & (norm[..., 2] >= -1.) & (norm[..., 2] <= 1.)
    return norm, valid2d, valid.float()


def frustum_to_voxel_forward(p, stereo_feat, stereo_feat_softmax, img_metas,
                             cur_sem_feats, coordinates_3d, depth_cfg,
                             sem_atten_feat=True, stereo_atten_feat=False,
                             cat_img_feature=True, num_3dconvs=1):
    """FrustumToVoxel.forward, feature_transformation.py:68-173 (batch loop
    included; like the reference, pad_shape is read from img_metas[0])."""
    norms, v2ds, vs = [], [], []
    for m in img_metas:
        n, v2, v = frustum_grid(coordinates_3d, m['cam2img'],
                                img_metas[0]['pad_shape'], depth_cfg)
        norms.append(n)
        v2ds.append(v2)
        vs.append(v)
    # the fp32 geometry is built on the CPU; widened exactly for fp64 features
    norm = torch.stack(norms).to(stereo_feat)
    valid2d = torch.stack(v2ds).to(stereo_feat.device)
    valid = torch.stack(vs).to(stereo_feat.device)
    voxel = F.grid_sample(stereo_feat, norm, align_corners=True)
    voxel = voxel * valid[:, None]
    pred_disp = None
    if stereo_atten_feat or (sem_atten_feat and cat_img_feature):
        pred_disp = F.grid_sample(stereo_feat_softmax, norm, align_corners=True)
        pred_disp = pred_disp * valid[:, None]
        if stereo_atten_feat:
            voxel = voxel * pred_disp
    if cat_img_feature:
        norm2d = norm.clone()
        norm2d[..., 2] = 0
        v2 = F.grid_sample(cur_sem_feats.unsqueeze(2), norm2d, align_corners=True)
        v2 = v2 * valid2d.float()[:, None]
        if sem_atten_feat:
            v2 = v2 * pred_disp
        voxel = torch.cat([voxel, v2], dim=1)
    for i in range(num_3dconvs):
        voxel = _conv_module(voxel, p, f'voxel_convs.{i}.0')
    return F.avg_pool3d(voxel, (4, 1, 1), stride=(4, 1, 1))


# ----------------------------------------------------------------------------
# f3  BEVHourglass + LIGAAnchor3DHead.forward (SURVEY.md section 8(f) row 3): the 2-D
# stage that turns the voxel features into class scores and 3-D box regressions
# ----------------------------------------------------------------------------
def _gn2d(x, p, prefix, groups=32):
    return F.group_norm(x, groups, p[prefix + '.weight'], p[prefix + '.bias'], GN_EPS)


def bev_hourglass_forward(p, spatial_features):
    """BEVHourglass.forward with norm_cfg GN (backbones/bev_hourglass.py:39-50) and
    hourglass2d.forward (:121-137) with presqu = postsqu = None; convbn = Conv2d(bias=False) +
    GroupNorm(32) (models/utils/conv_modules.py:6-24).  Returns (prehg, spatial_features_2d)."""
    x = F.relu(_gn2d(F.conv2d(spatial_features, p['compress_conv.conv.weight'], None, 1, 1),
                     p, 'compress_conv.gn'))                                   # :40
    hg = 'bev_hourglass.'
    out = F.relu(_gn2d(F.conv2d(x, p[hg + 'conv1.0.0.weight'], None, 2, 1),
                       p, hg + 'conv1.0.1'))                                   # :122
    pre = F.relu(_gn2d(F.conv2d(out, p[hg + 'conv2.0.weight'], None, 1, 1),
                       p, hg + 'conv2.1'))                                     # :123-127
    out = F.relu(_gn2d(F.conv2d(pre, p[hg + 'conv3.0.0.weight'], None, 2, 1),
                       p, hg + 'conv3.0.1'))                                   # :129
    out = F.relu(_gn2d(F.conv2d(out, p[hg + 'conv4.0.0.weight'], None, 1, 1),
                       p, hg + 'conv4.0.1'))                                   # :130
    post = F.relu(_gn2d(F.conv_transpose2d(out, p[hg + 'conv5.0.weight'], None, 2, 1, 1),
                        p, hg + 'conv5.1') + pre)                              # :135
    out = _gn2d(F.conv_transpose2d(post, p[hg + 'conv6.0.weight'], None, 2, 1, 1),
                p, hg + 'conv6.1')                                             # :137
    return x, out                                                              # :47-48


def liga_anchor3d_head_forward(p, x, num_convs=2):
    """LIGAAnchor3DHead.forward_single (dense_heads/liga_anchor3d_head.py:108-128) with the
    layers of _init_layers (:37-75): num_convs x ConvModule(3x3, GN, ReLU) per branch, 3x3
    conv_cls / conv_reg with bias, 1x1 conv_dir_cls on the CLASSIFICATION features."""
    cls_feats = reg_feats = x
    for i in range(num_convs):
        cls_feats = F.relu(_gn2d(F.conv2d(cls_feats, p[f'cls_convs.{i}.conv.weight'], None, 1, 1),
                                 p, f'cls_convs.{i}.gn'))
        reg_feats = F.relu(_gn2d(F.conv2d(reg_feats, p[f'reg_convs.{i}.conv.weight'], None, 1, 1),
                                 p, f'reg_convs.{i}.gn'))
    cls_score = F.conv2d(cls_feats, p['conv_cls.weight'], p['conv_cls.bias'], 1, 1)
    bbox_pred = F.conv2d(reg_feats, p['conv_reg.weight'], p['conv_reg.bias'], 1, 1)
    dir_cls_preds = F.conv2d(cls_feats, p['conv_dir_cls.weight'], p['conv_dir_cls.bias'])
    return cls_score, bbox_pred, dir_cls_preds


def dfm_bev_stage(p_bev, p_head, volume_feat, num_convs=2):
    """DfM.simple_test after feature_transformation (detectors/dfm.py:426-432): height
    compression view, backbone_3d, bbox_head_3d([bev_feat]) -> (cls_score, bbox_pred,
    dir_cls_preds) of the single level."""
    _, cv, nz, ny, nx = volume_feat.shape
    bev_feat = volume_feat.reshape(-1, cv * nz, ny, nx)
    _, bev = bev_hourglass_forward(p_bev, bev_feat)
    return liga_anchor3d_head_forward(p_head, bev, num_convs)


def bf16_round(x):
    """Round-to-nearest-even to bf16 precision, kept in fp32 (precision study only)."""
    return x.to(torch.bfloat16).to(torch.float32)


# ----------------------------------------------------------------------------
# f2  SPPUNetNeck tail (SURVEY.md section 8(f) row 2): the last two layers that produce the
# full-resolution 32-channel stereo feature build_dfm_cost consumes
# ----------------------------------------------------------------------------
def spp_unet_lastconv(p, x):
    """SPPUNetNeck.lastconv (necks/spp_unet_neck.py:60-75, applied at :110):
    ConvModule(3x3, GN(32), ReLU) then Conv2d(1x1, bias=False)."""
    y = F.relu(_gn2d(F.conv2d(x, p['lastconv.0.conv.weight'], None, 1, 1), p, 'lastconv.0.gn'))
    return F.conv2d(y, p['lastconv.1.weight'])


def tf32_round(x):
    """Round-to-nearest-even to 10 mantissa bits (precision study only)."""
    xi = x.contiguous().view(torch.int32)
    r = ((xi >> 13) & 1) + 0x0FFF
    return ((xi + r) & ~0x1FFF).view(torch.float32)
