"""Deterministic synthetic inputs for tests and bench (SURVEY.md section 8d).

There is no dataset or checkpoint on the GPU box, so the workload is: smooth
(band-limited) random 32-channel stereo features at the KITTI shape, the real
KITTI demo-sample geometry (numbers below were read once from the reference's
``demo/data/kitti/kitti_000008_infos.pkl``: ``P2`` and
``inv(prev_cam2global) @ cur_cam2global`` as ``VideoPipeline`` derives it,
mmdet3d/datasets/pipelines/loading.py:530-537), and random weights keyed by the
reference ``state_dict`` names.  Everything is generated from NumPy's legacy
MT19937 ``RandomState`` so every process regenerates identical tensors.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# KITTI sample 000008, camera 2 projection padded to 4x4 (calib['P2'])
KITTI_P2 = np.array(
    [[721.5377, 0.0, 609.5593, 44.85728],
     [0.0, 721.5377, 172.854, 0.2163791],
     [0.0, 0.0, 1.0, 0.002745884],
     [0.0, 0.0, 0.0, 1.0]], dtype=np.float64)

# cur -> prev camera transforms for the three previous sweeps of the demo sample
KITTI_CUR2PREV = np.array([
    [[0.999302046, -0.001022011, 0.037342192, 0.048377033],
     [0.000957212, 0.99999813, 0.00173758, 0.015017807],
     [-0.037344459, -0.001701675, 0.999300674, 0.321288688],
     [0.0, 0.0, 0.0, 1.0]],
    [[0.99658589, -0.004466793, 0.082434821, 0.122045509],
     [0.004160789, 0.999984333, 0.003887874, 0.034121847],
     [-0.082450365, -0.003532619, 0.996588961, 0.662983686],
     [0.0, 0.0, 0.0, 1.0]],
    [[0.991866141, -0.009969419, 0.126890392, 0.213423159],
     [0.009329447, 0.999941439, 0.005634116, 0.059576494],
     [-0.126938255, -0.004405767, 0.991900695, 0.958234025],
     [0.0, 0.0, 0.0, 1.0]]], dtype=np.float64)


def depth_cfg_for(num_planes, downsample_factor=4):
    """Model-level depth_cfg (configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:4-9)
    with num_bins chosen so that D = num_bins / downsample_factor planes."""
    return dict(mode='UD', num_bins=num_planes * downsample_factor,
                depth_min=2, depth_max=59.6,
                downsample_factor=downsample_factor)


def smooth_field(rng, c, h, w, cell=8):
    """Band-limited random feature map [1, c, h, w] fp32 (N(0,1) on a 1/cell
    lattice, bicubic-upsampled) -- bilinear taps of it are not noise-amplifying
    (SURVEY.md section 7, 'sampling-coordinate reproducibility')."""
    lh, lw = math.ceil(h / cell) + 3, math.ceil(w / cell) + 3
    low = torch.from_numpy(
        rng.standard_normal((1, c, lh, lw)).astype(np.float32))
    up = F.interpolate(low, size=(lh * cell, lw * cell), mode='bicubic',
                       align_corners=False)
    return up[:, :, cell:cell + h, cell:cell + w].contiguous()


def make_img_meta(h, w, sweep=2, flip=False, crop_offset=(0, 0), scale=1.0,
                  ori_shape=None):
    """The img_meta keys DfMBackbone.forward reads (dfm_backbone.py:150-172)."""
    if ori_shape is None:
        ori_shape = (h, w, 3)
    return dict(
        ori_cam2img=KITTI_P2.astype(np.float32).tolist(),
        cur2prevs=torch.from_numpy(
            KITTI_CUR2PREV[sweep:sweep + 1].astype(np.float32)),
        ori_shape=tuple(ori_shape),
        pad_shape=(h, w, 3),
        img_shape=(h, w, 3),
        flip=flip,
        crop_offset=list(crop_offset),
        scale_factor=[scale, scale, scale, scale])


def kitti_p2_for_width(w):
    """KITTI P2 with its focal lengths and principal point rescaled to an image w pixels wide
    (w = 1248 keeps the whole lattice of a w-wide feature map inside the original field of
    view at the demo sample's scale)."""
    p = KITTI_P2.copy()
    p[:2] *= w / 1248.0
    return p


def cur2prev_pose(yaw=0.0, pitch=0.0, t=(0.0, 0.0, 0.0)):
    """A cur -> prev camera transform [4, 4] (camera axes: x right, y down, z forward):
    rotation by `yaw` about y, then `pitch` about x (radians), then translation t (metres)."""
    cy, sy = math.cos(yaw), math.sin(yaw)
    cp, sp = math.cos(pitch), math.sin(pitch)
    r_yaw = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    r_pitch = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    m = np.eye(4)
    m[:3, :3] = r_pitch @ r_yaw
    m[:3, 3] = t
    return m


def white_noise_pair(seed, c, h, w):
    """relu(N(0, 1)) (cur, prev) feature maps [1, c, h, w] fp32: neighbouring pixels differ by
    O(1), so a sample-coordinate error shows up undamped."""
    rng = np.random.RandomState(seed)
    return tuple(torch.from_numpy(rng.standard_normal((1, c, h, w)).astype(np.float32)).relu()
                 for _ in range(2))


def _kaiming(rng, shape, fan_in, gain=1.0):
    std = gain * math.sqrt(2.0 / fan_in)
    return (rng.standard_normal(shape) * std).astype(np.float32)


def make_backbone_params(rng, num_planes, in_channels=32, cv=32):
    """Random DfMBackbone parameters keyed by the reference state_dict names
    (SURVEY.md section 8a 'State').  GroupNorm affine is randomised so gamma/beta
    are exercised."""
    p = {}

    def gn(name, c):
        p[name + '.weight'] = (0.5 + rng.random_sample(c)).astype(np.float32)
        p[name + '.bias'] = (0.2 * rng.standard_normal(c)).astype(np.float32)

    def convmod(name, cin, cout):
        p[name + '.conv.weight'] = _kaiming(rng, (cout, cin, 3, 3, 3), cin * 27)
        gn(name + '.gn', cout)

    def hg(name, c):
        for sub, ci, co, seq in (('conv1', c, 2 * c, True),
                                 ('conv2', 2 * c, 2 * c, False),
                                 ('conv3', 2 * c, 2 * c, True),
                                 ('conv4', 2 * c, 2 * c, True)):
            pre = f'{name}.{sub}.0' if seq else f'{name}.{sub}'
            p[pre + '.0.weight'] = _kaiming(rng, (co, ci, 3, 3, 3), ci * 27)
            gn(pre + '.1', co)
        # ConvTranspose3d weight layout is (in, out, kd, kh, kw)
        p[f'{name}.conv5.0.weight'] = _kaiming(
            rng, (2 * c, 2 * c, 3, 3, 3), 2 * c * 27 / 8)
        gn(f'{name}.conv5.1', 2 * c)
        p[f'{name}.conv6.0.weight'] = _kaiming(
            rng, (2 * c, c, 3, 3, 3), 2 * c * 27 / 8)
        gn(f'{name}.conv6.1', c)

    for sfx, cin in (('', 2 * in_channels), ('_mono', in_channels)):
        convmod('dres0' + sfx, cin, cv)
        convmod('dres1' + sfx, cv, cv)
        tower = 'mono' if sfx else 'stereo'
        hg(f'hg_{tower}.0', cv)
        convmod(f'pred_{tower}.0.0', cv, cv)
        p[f'pred_{tower}.0.1.weight'] = _kaiming(rng, (1, cv, 3, 3, 3), cv * 27)
    p['aggregate_cost.weight'] = _kaiming(
        rng, (num_planes, 2 * num_planes, 1, 1), 2 * num_planes, gain=0.7)
    return {k: torch.from_numpy(v) for k, v in p.items()}


def make_kitti_pair(seed, h, w, num_planes, c=32, sweep=2, flip=False,
                    crop_offset=(0, 0), scale=1.0, ori_shape=None):
    """One synthetic (cur, prev) stereo-feature pair + img_metas + weights."""
    rng = np.random.RandomState(seed)
    cur = smooth_field(rng, c, h, w)
    prev = smooth_field(rng, c, h, w)
    params = make_backbone_params(rng, num_planes, c, 32)
    metas = [make_img_meta(h, w, sweep, flip, crop_offset, scale, ori_shape)]
    return cur, prev, metas, params


def make_neck_params(rng, template_state_dict):
    """Random DfMNeck / OutdoorImVoxelNeck parameters shaped like (and ordered as)
    ``template_state_dict``; BatchNorm running statistics are randomised so the
    eval-mode affine is exercised (SURVEY.md section 8d)."""
    out = {}
    for k, v in template_state_dict.items():
        shape = tuple(v.shape)
        if k.endswith('num_batches_tracked'):
            out[k] = torch.zeros(shape, dtype=v.dtype)
        elif k.endswith('conv.weight'):
            fan_in = shape[1] * 27
            out[k] = torch.from_numpy(_kaiming(rng, shape, fan_in))
        elif k.endswith('aggregate_layer.weight'):
            out[k] = torch.from_numpy(_kaiming(rng, shape, shape[1], gain=0.5))
        elif k.endswith('bn.weight'):
            out[k] = torch.from_numpy(
                (0.5 + rng.random_sample(shape)).astype(np.float32))
        elif k.endswith('bn.bias') or k.endswith('running_mean'):
            out[k] = torch.from_numpy(
                (0.2 * rng.standard_normal(shape)).astype(np.float32))
        elif k.endswith('running_var'):
            out[k] = torch.from_numpy(
                (0.5 + rng.random_sample(shape)).astype(np.float32))
        else:
            raise KeyError(k)
    return out


# KITTI model-level voxel grid (configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:1,10-11)
KITTI_POINT_CLOUD_RANGE = [2, -30.4, -3, 59.6, 30.4, 1]
KITTI_VOXEL_SIZE = [0.2, 0.2, 0.2]


def frustum_voxel_centres(point_cloud_range, n_voxels):
    """The three axes of ``DfM.prepare_coordinates_3d`` (detectors/dfm.py:193-211):
    linspace of voxel centres, (nx, ny, nz) cells."""
    pcr = point_cloud_range
    axes = []
    for a, n in enumerate(n_voxels):
        vs = (pcr[3 + a] - pcr[a]) / n
        axes.append(torch.linspace(pcr[a] + vs / 2., pcr[3 + a] - vs / 2., n,
                                   dtype=torch.float32))
    return axes


def frustum_coordinates(point_cloud_range, n_voxels):
    """coordinates_3d [nz, ny, nx, 3] holding (x, y, z), detectors/dfm.py:208-211."""
    xs, ys, zs = frustum_voxel_centres(point_cloud_range, n_voxels)
    zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing='ij')
    return torch.stack([xx, yy, zz], dim=-1).float()


def make_frustum_case(seed, h, w, num_planes, n_voxels, num_3dconvs=1,
                      cat_img_feature=True):
    """Synthetic FrustumToVoxel inputs: ``h x w`` is the padded network input,
    the plane-sweep volume is [32, num_planes, h/4, w/4].  cam2img is KITTI P2
    rescaled to the h x w image so that part of the grid projects outside."""
    rng = np.random.RandomState(seed)
    ho, wo = h // 4, w // 4
    stereo = torch.cat([smooth_field(rng, 32, ho, wo, cell=4)
                        for _ in range(num_planes)], 0)
    stereo = stereo.permute(1, 0, 2, 3)[None].contiguous()  # [1,32,D,ho,wo]
    cost = torch.cat([smooth_field(rng, 1, ho, wo, cell=4)
                      for _ in range(num_planes)], 1)[:, None] * 2.0
    sem = smooth_field(rng, 32, ho, wo, cell=4)
    s = w / 1248.0
    P = KITTI_P2.copy()
    P[:2] *= s
    P[1, 2] = 0.45 * h
    params = {}
    cin = 64 if cat_img_feature else 32
    for i in range(num_3dconvs):
        ci = cin if i == 0 else 32
        params[f'voxel_convs.{i}.0.conv.weight'] = torch.from_numpy(
            _kaiming(rng, (32, ci, 3, 3, 3), ci * 27))
        params[f'voxel_convs.{i}.0.gn.weight'] = torch.from_numpy(
            (0.5 + rng.random_sample(32)).astype(np.float32))
        params[f'voxel_convs.{i}.0.gn.bias'] = torch.from_numpy(
            (0.2 * rng.standard_normal(32)).astype(np.float32))
    metas = [dict(cam2img=P.astype(np.float32).tolist(), pad_shape=(h, w, 3))]
    return dict(stereo=stereo, cost=cost.contiguous(), sem=sem, metas=metas,
                params=params,
                coordinates_3d=frustum_coordinates(KITTI_POINT_CLOUD_RANGE,
                                                   n_voxels),
                depth_cfg=depth_cfg_for(num_planes))


# Waymo multi-view workload (configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync
# [_10sweeps].py: input 832x1248 after MultiViewImageResize3D, FPN level-0 features at stride 4,
# n_voxels [220, 300, 12] over [-35, -75, -2, 75, 75, 4]; detectors/multiview_dfm.py:54-61)
WAYMO_N_VOXELS = [220, 300, 12]
WAYMO_RANGE = [-35.0, -75.0, -2.0, 75.0, 75.0, 4.0]
WAYMO_INPUT_HW = (832, 1248)
WAYMO_FEAT_HW = (208, 312)


def waymo_lidar2img(num_frames, num_views=5, ego_shift=1.0):
    """Synthetic pinhole rig: cameras yawed over the front half-circle, focal length
    2055 px * 0.65 (resize), principal point at the image centre; earlier frames are
    shifted `ego_shift` metres backwards.  [T*Nv, 4, 4] float64."""
    mats = []
    for f in range(num_frames):
        for v in range(num_views):
            yaw = (v - (num_views - 1) / 2) * 0.7
            r = np.array([[np.cos(yaw), np.sin(yaw), 0], [-np.sin(yaw), np.cos(yaw), 0],
                          [0, 0, 1]])
            # lidar (x fwd, y left, z up) -> camera (x right, y down, z fwd)
            l2c = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64) @ r
            ext = np.eye(4)
            ext[:3, :3] = l2c
            ext[:3, 3] = l2c @ np.array([-ego_shift * f, 0.03 * v, -1.5])
            k = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0],
                          [0, 0, 0, 1]])
            mats.append(k @ ext)
    return np.array(mats)


def make_waymo_sample(seed, num_frames, num_views=5, channels=64, feat_hw=WAYMO_FEAT_HW,
                      input_hw=WAYMO_INPUT_HW, flip=False, scale=1.0, crop=(0.0, 0.0)):
    """One sample of MultiViewDfM.feature_transformation's inputs: [T*Nv, C, Hf, Wf] features
    and the img_meta keys multiview_dfm.py:139-170 reads."""
    rng = np.random.RandomState(seed)
    s = num_frames * num_views
    feats = torch.from_numpy(
        rng.standard_normal((s, channels) + tuple(feat_hw)).astype(np.float32))
    meta = dict(ori_lidar2img=waymo_lidar2img(num_frames, num_views),
                input_shape=tuple(input_hw),
                img_shape=[(input_hw[0], input_hw[1], 3)] * s,
                scale_factor=np.array([scale, scale, scale, scale], dtype=np.float32),
                img_crop_offset=list(crop), flip=flip, num_views=num_views,
                num_ref_frames=num_frames - 1)
    return feats, meta


def make_bev_params(rng, in_channels=160, c=64):
    """Random BEVHourglass parameters keyed like the reference state_dict
    (backbones/bev_hourglass.py:25-32, 53-119; GroupNorm variant of the KITTI config)."""
    p = {}

    def gn(name, ch):
        p[name + '.weight'] = (0.5 + rng.random_sample(ch)).astype(np.float32)
        p[name + '.bias'] = (0.2 * rng.standard_normal(ch)).astype(np.float32)

    p['compress_conv.conv.weight'] = _kaiming(rng, (c, in_channels, 3, 3), in_channels * 9)
    gn('compress_conv.gn', c)
    hg = 'bev_hourglass.'
    for sub, ci, co, seq in (('conv1', c, 2 * c, True), ('conv2', 2 * c, 2 * c, False),
                             ('conv3', 2 * c, 2 * c, True), ('conv4', 2 * c, 2 * c, True)):
        pre = f'{hg}{sub}.0' if seq else f'{hg}{sub}'
        p[pre + '.0.weight'] = _kaiming(rng, (co, ci, 3, 3), ci * 9)
        gn(pre + '.1', co)
    p[hg + 'conv5.0.weight'] = _kaiming(rng, (2 * c, 2 * c, 3, 3), 2 * c * 9 / 4)  # (in, out, k, k)
    gn(hg + 'conv5.1', 2 * c)
    p[hg + 'conv6.0.weight'] = _kaiming(rng, (2 * c, c, 3, 3), 2 * c * 9 / 4)
    gn(hg + 'conv6.1', c)
    return {k: torch.from_numpy(v) for k, v in p.items()}


def make_anchor_head_params(rng, c=64, num_convs=2, num_anchors=6, num_classes=3,
                            box_code_size=7):
    """Random LIGAAnchor3DHead parameters (dense_heads/liga_anchor3d_head.py:37-75): 6 anchors
    (3 classes x 2 rotations, KITTI config) -> 18 class / 42 box / 12 direction channels."""
    p = {}
    for br in ('cls_convs', 'reg_convs'):
        for i in range(num_convs):
            p[f'{br}.{i}.conv.weight'] = _kaiming(rng, (c, c, 3, 3), c * 9)
            p[f'{br}.{i}.gn.weight'] = (0.5 + rng.random_sample(c)).astype(np.float32)
            p[f'{br}.{i}.gn.bias'] = (0.2 * rng.standard_normal(c)).astype(np.float32)
    for name, co, k in (('conv_cls', num_anchors * num_classes, 3),
                        ('conv_reg', num_anchors * box_code_size, 3),
                        ('conv_dir_cls', num_anchors * 2, 1)):
        p[name + '.weight'] = _kaiming(rng, (co, c, k, k), c * k * k, gain=0.7)
        p[name + '.bias'] = (0.1 * rng.standard_normal(co)).astype(np.float32)
    return {k: torch.from_numpy(v) for k, v in p.items()}


BEV_CASE = dict(seed=91, nz=5, ny=44, nx=36)   # 3 x 5 tiles of the 16 x 8 conv tile, ragged


def make_bev_case(seed=91, nz=5, ny=44, nx=36, cv=32):
    """volume_feat [1, cv, nz, ny, nx] (what FrustumToVoxel returns) + parameters of the 2-D
    stage; the KITTI config has nz=5, ny=304, nx=288."""
    rng = np.random.RandomState(seed)
    vol = torch.from_numpy(rng.standard_normal((1, cv, nz, ny, nx)).astype(np.float32)).relu()
    return dict(volume=vol, bev=make_bev_params(rng, cv * nz), head=make_anchor_head_params(rng))


# the Anchor3DHead fixture (tests/golden/anchor3d_head.npz): 37 x 29 = 1,073 cells, i.e. 8 full
# 128-cell tiles of the 1x1-conv kernel plus a ragged tail of 49
ANCHOR3D_HEAD_CASE = dict(seed=101, feat=256, ny=37, nx=29)


def make_anchor3d_head_case(seed=101, feat=256, ny=37, nx=29, num_anchors=6, num_classes=3,
                            box_code_size=7):
    """Inputs of the Anchor3DHead fixture: random (not near-zero-init) parameters of the three
    1x1 convs in the reference state_dict order (dense_heads/anchor3d_head.py:139-147), and a
    non-negative BEV map x [1, feat, ny, nx] (the neck's output is a blend of ReLUs)."""
    rng = np.random.RandomState(seed)
    p = {}
    for name, co in (('conv_cls', num_anchors * num_classes),
                     ('conv_reg', num_anchors * box_code_size),
                     ('conv_dir_cls', num_anchors * 2)):
        p[name + '.weight'] = (rng.standard_normal((co, feat, 1, 1)) /
                               np.sqrt(feat)).astype(np.float32)
        p[name + '.bias'] = (0.1 * rng.standard_normal(co)).astype(np.float32)
    a = np.maximum(rng.standard_normal((1, feat, ny, nx)), 0)
    b = np.maximum(rng.standard_normal((1, feat, ny, nx)), 0)
    x = torch.from_numpy((0.7 * a + 0.3 * b).astype(np.float32))
    return x, {k: torch.from_numpy(v) for k, v in p.items()}


# SPPUNetNeck of the shipped KITTI config (configs/dfm/dfm_r34_1x8_kitti-3d-3class.py `neck`):
# state_dict entries in the reference order (necks/spp_unet_neck.py:35-91,
# models/utils/conv_modules.py:46-60)
def spp_neck_state_shapes():
    shapes = []
    for i in range(4):
        p = f'spp_branches.{i}.1.'
        shapes += [(p + 'conv.weight', (32, 128, 1, 1)), (p + 'gn.weight', (32,)),
                   (p + 'gn.bias', (32,))]
    for name, (co, ci) in (('conv.0', (64, 512)), ('conv.1', (32, 64)),
                           ('redir.0', (64, 64)), ('redir.1', (32, 3))):
        p = f'upconv_module.{name}.'
        shapes.append((p + '0.weight', (co, ci, 3, 3)))
        shapes += [(p + '1.' + f, (co,)) for f in ('weight', 'bias', 'running_mean',
                                                   'running_var')]
        shapes.append((p + '1.num_batches_tracked', ()))
    shapes += [('lastconv.0.conv.weight', (32, 32, 3, 3)), ('lastconv.0.gn.weight', (32,)),
               ('lastconv.0.gn.bias', (32,)), ('lastconv.1.weight', (32, 32, 1, 1))]
    for i, (co, ci) in enumerate(((128, 512), (32, 128))):
        p = f'rpnconv.{i}.'
        shapes += [(p + 'conv.weight', (co, ci, 3, 3)), (p + 'gn.weight', (co,)),
                   (p + 'gn.bias', (co,))]
    return shapes


def make_spp_neck_case(seed, H, W):
    """Inputs of SPPUNetNeck at image size H x W: feats = [img, f1, f2, f3, f4] ([1, C, h, w]
    smooth fields with LIGAResNet34's shapes: 3 @ H, 64 @ H/2, 128 @ H/4 three times) and a random
    state_dict (reference keys and order): Kaiming weights, GN / BN affines around 1 / 0, BN
    running statistics away from the identity, so every folded affine carries signal."""
    rng = np.random.RandomState(seed)
    feats = [smooth_field(rng, 3, H, W, cell=16),
             smooth_field(rng, 64, H // 2, W // 2)]
    feats += [torch.relu(smooth_field(rng, 128, H // 4, W // 4, cell=4)) for _ in range(3)]
    sd = {}
    for k, shape in spp_neck_state_shapes():
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif len(shape) == 4:
            sd[k] = torch.from_numpy(_kaiming(rng, shape, shape[1] * shape[2] * shape[3]))
        elif k.endswith('running_var'):
            sd[k] = torch.from_numpy((0.5 + rng.random_sample(shape)).astype(np.float32))
        elif k.endswith('running_mean'):
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
        elif k.endswith('weight'):
            sd[k] = torch.from_numpy((0.5 + rng.random_sample(shape)).astype(np.float32))
        else:
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
    return feats, sd


def liga_resnet_state_shapes():
    """(key, shape) of the reference LIGAResNet-34 state_dict of the KITTI config, in order
    (backbones/liga_resnet.py; mmdet ResLayer naming, BatchNorm statistics included)."""
    def bn(prefix, c):
        return [(prefix + f, (c,)) for f in ('.weight', '.bias', '.running_mean', '.running_var')] + \
            [(prefix + '.num_batches_tracked', ())]
    shapes = [('conv1.weight', (64, 3, 7, 7))] + bn('bn1', 64)
    inplanes = 64
    for s, (n, planes) in enumerate(zip((3, 4, 6, 3), (64, 128, 128, 128))):
        for j in range(n):
            p = f'layer{s + 1}.{j}.'
            shapes += [(p + 'conv1.weight', (planes, inplanes, 3, 3))] + bn(p + 'bn1', planes)
            shapes += [(p + 'conv2.weight', (planes, planes, 3, 3))] + bn(p + 'bn2', planes)
            if j == 0 and inplanes != planes:
                shapes += [(p + 'downsample.0.weight', (planes, inplanes, 1, 1))] + \
                    bn(p + 'downsample.1', planes)
            inplanes = planes
    return shapes


def make_liga_resnet_case(seed, H, W, B=1):
    """Inputs of LIGAResNet at image size H x W: a normalised-image-like batch [B, 3, H, W]
    (smooth fields) and a random state_dict (reference keys and order): Kaiming conv weights,
    BatchNorm statistics away from the identity; bn2's gamma is kept below 1 so the 16-block
    residual chain (no ReLU after the adds) stays O(1)."""
    rng = np.random.RandomState(seed)
    img = torch.cat([smooth_field(rng, 3, H, W, cell=4) for _ in range(B)], 0)
    sd = {}
    for k, shape in liga_resnet_state_shapes():
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif len(shape) == 4:
            sd[k] = torch.from_numpy(_kaiming(rng, shape, shape[1] * shape[2] * shape[3]))
        elif k.endswith('running_var'):
            sd[k] = torch.from_numpy((0.5 + rng.random_sample(shape)).astype(np.float32))
        elif k.endswith('running_mean'):
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
        elif k.endswith('weight'):
            lo, hi = (0.2, 0.6) if '.bn2.' in k or 'downsample.1' in k else (0.5, 1.5)
            sd[k] = torch.from_numpy((lo + (hi - lo) * rng.random_sample(shape)).astype(np.float32))
        else:
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
    return img, sd


def resnet101_state_shapes():
    """(key, shape) of mmdet's ResNet-101 state_dict with DCNv2 in layer3 / layer4 (the Waymo
    configs' backbone), in order: 676 entries, BatchNorm statistics and conv_offset included."""
    def bn(prefix, c):
        return [(prefix + f, (c,)) for f in ('.weight', '.bias', '.running_mean', '.running_var')] + \
            [(prefix + '.num_batches_tracked', ())]
    shapes = [('conv1.weight', (64, 3, 7, 7))] + bn('bn1', 64)
    inplanes = 64
    for s, n in enumerate((3, 4, 23, 3)):
        planes = 64 << s
        for j in range(n):
            p = f'layer{s + 1}.{j}.'
            shapes += [(p + 'conv1.weight', (planes, inplanes, 1, 1))] + bn(p + 'bn1', planes)
            shapes.append((p + 'conv2.weight', (planes, planes, 3, 3)))
            if s >= 2:
                shapes += [(p + 'conv2.conv_offset.weight', (27, planes, 3, 3)),
                           (p + 'conv2.conv_offset.bias', (27,))]
            shapes += bn(p + 'bn2', planes)
            shapes += [(p + 'conv3.weight', (4 * planes, planes, 1, 1))] + bn(p + 'bn3', 4 * planes)
            if j == 0:
                shapes += [(p + 'downsample.0.weight', (4 * planes, inplanes, 1, 1))] + \
                    bn(p + 'downsample.1', 4 * planes)
            inplanes = 4 * planes
    return shapes


def make_resnet101_case(seed, H, W, B=1):
    """Inputs of the Waymo ResNet-101 + DCNv2 backbone at image size H x W: a
    normalised-image-like batch [B, 3, H, W] (smooth fields) and a random state_dict (mmdet's
    keys and order).  Kaiming conv weights; BatchNorm statistics away from the identity; bn3 and
    the downsample's gamma small (0.1 - 0.3) so the 33-block residual chain stays O(1).  mmcv
    zero-initialises conv_offset, which would reduce every DCN to a plain conv times 0.5; here
    its weights give offsets of several pixels (samples leave the map, a few land near integer
    positions) and its bias spreads the masks over (0, 1)."""
    rng = np.random.RandomState(seed)
    img = torch.cat([smooth_field(rng, 3, H, W, cell=4) for _ in range(B)], 0)
    sd = {}
    for k, shape in resnet101_state_shapes():
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif 'conv_offset' in k:
            # the input of conv_offset is a ReLU'd, BN'd activation of O(1): offsets of a few
            # pixels for gain ~3 (the 27 channels of a tap share no scale)
            a = _kaiming(rng, shape, shape[1] * 9, gain=2.0) if len(shape) == 4 else \
                (np.concatenate([1.5 * rng.standard_normal(18),
                                 rng.standard_normal(9)]).astype(np.float32))
            sd[k] = torch.from_numpy(a)
        elif len(shape) == 4:
            sd[k] = torch.from_numpy(_kaiming(rng, shape, shape[1] * shape[2] * shape[3]))
        elif k.endswith('running_var'):
            sd[k] = torch.from_numpy((0.5 + rng.random_sample(shape)).astype(np.float32))
        elif k.endswith('running_mean'):
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
        elif k.endswith('weight'):
            lo, hi = (0.1, 0.3) if '.bn3.' in k or 'downsample.1' in k else (0.5, 1.5)
            sd[k] = torch.from_numpy((lo + (hi - lo) * rng.random_sample(shape)).astype(np.float32))
        else:
            sd[k] = torch.from_numpy((0.2 * rng.standard_normal(shape)).astype(np.float32))
    return img, sd


# ---- anchor-head post-processing (get_bboxes) ----

KITTI_ANCHOR_GENERATOR = dict(   # configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:160-167
    type='Anchor3DRangeGenerator',
    ranges=[[2, -30.4, -1.78, 59.6, 30.4, -1.78], [2, -30.4, -0.6, 59.6, 30.4, -0.6],
            [2, -30.4, -0.6, 59.6, 30.4, -0.6]],
    sizes=[[3.9, 1.6, 1.56], [0.8, 0.6, 1.73], [1.76, 0.6, 1.73]],
    rotations=[0, 1.57], reshape_out=False)
WAYMO_ANCHOR_GENERATOR = dict(   # configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-*.py:41-53
    type='AlignedAnchor3DRangeGenerator',
    ranges=[[-35.0, -75.0, 0, 75.0, 75.0, 0], [-35.0, -75.0, -0.1188, 75.0, 75.0, -0.1188],
            [-35.0, -75.0, -0.0345, 75.0, 75.0, -0.0345]],
    sizes=[[0.91, 0.84, 1.74], [1.81, 0.84, 1.77], [4.73, 2.08, 1.77]],
    rotations=[0, 1.57], reshape_out=False)
KITTI_TEST_CFG = dict(use_rotate_nms=True, nms_across_levels=False, nms_thr=0.25,
                      score_thr=0.1, min_bbox_size=0, nms_pre=4096, max_num=500)
WAYMO_TEST_CFG = dict(use_rotate_nms=True, nms_across_levels=False, nms_thr=0.05,
                      score_thr=0.001, min_bbox_size=0, nms_pre=4096, max_num=500)
KITTI_DIR_OFFSET, WAYMO_DIR_OFFSET = 0.7854, -0.7854


def make_box_post_case(seed, ny, nx, num_anchors=6, ncol=3, num_objects=50, empty_class=None):
    """Synthetic head outputs (cls_score [A * ncol, ny, nx], bbox_pred [A * 7, ny, nx],
    dir_cls_preds [A * 2, ny, nx]) with `num_objects` planted objects: a 3 x 3-cell cluster whose
    anchors of one class carry logits of 1 .. 4 (kept below sigmoid saturation so scores rarely
    tie) and small varied deltas with an oblique yaw offset, so neighbouring boxes overlap and
    NMS suppresses heavily; on top of a background of logits around -4.  `empty_class` gets
    logits of -8 everywhere (no candidate at any shipped score_thr)."""
    rng = np.random.RandomState(seed)
    A = num_anchors
    cls = (-4.0 + 1.2 * rng.standard_normal((A, ncol, ny, nx))).astype(np.float32)
    box = (0.15 * rng.standard_normal((A, 7, ny, nx))).astype(np.float32)
    box[:, 6] = (0.4 * rng.standard_normal((A, ny, nx))).astype(np.float32)
    dirc = rng.standard_normal((A * 2, ny, nx)).astype(np.float32)
    for _ in range(num_objects):
        y, x = rng.randint(1, ny - 1), rng.randint(1, nx - 1)
        c = rng.randint(ncol if ncol < 4 else ncol - 1)
        yaw = rng.uniform(0.3, 1.3) * rng.choice([-1, 1])
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                for j in range(A):
                    cls[j, c, y + dy, x + dx] = rng.uniform(1.0, 4.0) - 0.3 * (abs(dx) + abs(dy))
                    box[j, :6, y + dy, x + dx] = 0.05 * rng.standard_normal(6)
                    box[j, 6, y + dy, x + dx] = yaw + 0.05 * rng.standard_normal()
    if empty_class is not None:
        cls[:, empty_class] = -8.0
    return (torch.from_numpy(cls.reshape(A * ncol, ny, nx)),
            torch.from_numpy(box.reshape(A * 7, ny, nx)), torch.from_numpy(dirc))


# name -> (generator, ny, nx, test_cfg, use_sigmoid, dir_offset, seed, extra case arguments)
BOX_POST_CASES = {
    'kitti_topk': (KITTI_ANCHOR_GENERATOR, 32, 24, dict(KITTI_TEST_CFG, nms_pre=2048), True,
                   KITTI_DIR_OFFSET, 301, dict(num_objects=12)),
    'waymo_no_topk': (WAYMO_ANCHOR_GENERATOR, 20, 16, WAYMO_TEST_CFG, True, WAYMO_DIR_OFFSET,
                      302, dict(num_objects=8)),
    'kitti_max_num_empty_class': (KITTI_ANCHOR_GENERATOR, 24, 20,
                                  dict(KITTI_TEST_CFG, nms_pre=1500, max_num=20), True,
                                  KITTI_DIR_OFFSET, 303, dict(num_objects=14, empty_class=2)),
    'waymo_softmax': (WAYMO_ANCHOR_GENERATOR, 16, 12, dict(WAYMO_TEST_CFG, nms_pre=600,
                                                           score_thr=0.05), False,
                      WAYMO_DIR_OFFSET, 304, dict(num_objects=6, ncol=4)),
}


def _max_iou_assigner(pos, neg):
    return dict(type='MaxIoUAssigner', iou_calculator=dict(type='BboxOverlapsNearest3D'),
                pos_iou_thr=pos, neg_iou_thr=neg, min_pos_iou=neg, ignore_iof_thr=-1)


# train_cfg and loss settings of the shipped heads (configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:
# 151-225, configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py:35-92)
KITTI_TRAIN_CFG = dict(assigner=[_max_iou_assigner(0.6, 0.45), _max_iou_assigner(0.5, 0.35),
                                 _max_iou_assigner(0.5, 0.35)],
                       allowed_border=0, pos_weight=-1, debug=False)
WAYMO_TRAIN_CFG = dict(assigner=[_max_iou_assigner(0.5, 0.35), _max_iou_assigner(0.5, 0.35),
                                 _max_iou_assigner(0.6, 0.45)],
                       allowed_border=0, pos_weight=-1, debug=False)
FOCAL_LOSS = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
KITTI_LOSSES = dict(loss_cls=FOCAL_LOSS,
                    loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5),
                    loss_dir=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=0.2),
                    loss_iou=dict(type='IOU3DLoss', loss_weight=1.0))
WAYMO_LOSSES = dict(loss_cls=FOCAL_LOSS,
                    loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=2.0),
                    loss_dir=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=0.2))


def make_anchor_loss_case(seed, anchors, ny, nx, num_sizes, num_rots, num_classes, num_gt,
                          drop_class=None, cross_class=False, head_scale=1.0):
    """Head outputs ([B, A * C, ny, nx], [B, A * 7, ny, nx], [B, A * 2, ny, nx]) and per-sample GT
    (``[M, 7]`` boxes, ``[M]`` int64 labels) for ``num_gt[b]`` boxes in sample b, planted on
    anchors of the table ``anchors`` [ny * nx * A, 7] (numpy fp32): jittered copies of random
    anchors, labelled by the anchor's size (a random class with ``cross_class``), plus, when a
    sample has at least 8, the edge cases: a GT equal to an anchor and its duplicate, yaws of
    exactly +-pi / 4 and beyond +-pi, and a box too small for any anchor to reach min_pos_iou.
    ``drop_class`` removes that class's GT (an assigner with no GT)."""
    rng = np.random.RandomState(seed)
    B, A, C = len(num_gt), num_sizes * num_rots, num_classes
    cls = (-2.0 + 1.5 * rng.standard_normal((B, A * C, ny, nx))) * head_scale
    box = 0.2 * rng.standard_normal((B, A * 7, ny, nx)) * head_scale
    dirc = rng.standard_normal((B, A * 2, ny, nx)) * head_scale
    gts, labels = [], []
    for m in num_gt:
        idx = rng.randint(0, anchors.shape[0], size=m)
        g = anchors[idx].astype(np.float64).copy()
        g[:, :2] += rng.uniform(-0.4, 0.4, (m, 2))
        g[:, 2] += rng.uniform(-0.2, 0.2, m)
        g[:, 3:6] *= rng.uniform(0.8, 1.25, (m, 3))
        g[:, 6] += 0.4 * rng.standard_normal(m)
        lab = (idx % A) // num_rots
        if cross_class:
            lab = rng.randint(0, C, size=m)
        if m >= 8:
            g[0] = anchors[idx[0]]
            g[1] = g[0]
            lab[1] = lab[0]
            g[2, 6], g[3, 6] = np.float32(np.pi / 4), -np.float32(np.pi / 4)
            g[4, 6], g[5, 6] = np.pi + 0.3, -np.pi - 0.4
            g[6, 3:6] = 0.08
        g = g.astype(np.float32)
        keep = lab != drop_class if drop_class is not None else np.ones(m, bool)
        gts.append(torch.from_numpy(g[keep]))
        labels.append(torch.from_numpy(lab[keep].astype(np.int64)))
    t = lambda a: torch.from_numpy(a.astype(np.float32))  # noqa: E731
    return t(cls), t(box), t(dirc), gts, labels


# name -> (head: 'liga' (KITTI config) or 'anchor3d' (Waymo config), ny, nx, GT per sample,
# make_anchor_loss_case arguments, LIGA's loss_iou on, seed): tests/golden/anchor_loss.npz
ANCHOR_LOSS_GOLDEN_CASES = {
    'liga_b1': ('liga', 40, 36, [20], {}, True, 401),
    'liga_b1_class_without_gt': ('liga', 40, 36, [16], dict(drop_class=2), True, 402),
    'liga_zero_positives': ('liga', 40, 36, [0], {}, False, 403),
    'liga_b2_one_empty': ('liga', 40, 36, [14, 0], {}, False, 404),
    'anchor3d_b1_cross_class': ('anchor3d', 30, 22, [60], dict(cross_class=True), False, 405),
    'anchor3d_b2': ('anchor3d', 30, 22, [40, 30], dict(cross_class=True), False, 406),
    'anchor3d_b2_one_empty': ('anchor3d', 30, 22, [0, 25], {}, False, 407),
}


def make_depth_loss_case(seed, n, D, H, W, f=4, density=0.05, num_boxes=6):
    """Inputs of ``DepthHead.loss`` for ``n`` images (B * N): smooth cost logits
    ``[n, 1, D, H, W]`` in about +-20 (``smooth_field``), a sparse scan-line-like depth map
    ``[n, fH, fW]`` and int32 foreground masks of box ids + 1 (0 = background), as the
    training pipeline gives them.  Rows are LiDAR scan lines; about ``density`` of the pixels
    carry a depth, drawn uniformly over [0, 65] so some fall outside the shipped [2, 59.6]
    range.  The density is a synthetic choice, not a measured KITTI figure; 1.0 gives every
    pixel a depth."""
    rng = np.random.RandomState(seed)
    fh, fw = f * H, f * W
    cost = torch.stack([7.0 * smooth_field(rng, D, H, W, cell=4)[0] for _ in range(n)])[:, None]
    row_p = min(1.0, 4.0 * density)
    rows = rng.uniform(size=(n, fh, 1)) < row_p
    cols = rng.uniform(size=(n, fh, fw)) < density / row_p
    depth = rng.uniform(0.0, 65.0, size=(n, fh, fw)).astype(np.float32)
    depth = np.where(rows & cols, depth, np.float32(0.0))
    fg = np.zeros((n, fh, fw), np.int32)
    for i in range(n):
        for b in range(num_boxes):
            y0, x0 = rng.randint(0, fh), rng.randint(0, fw)
            bh, bw = rng.randint(1, max(2, fh // 3)), rng.randint(1, max(2, fw // 4))
            fg[i, y0:y0 + bh, x0:x0 + bw] = b + 1
    return cost.contiguous(), torch.from_numpy(depth), torch.from_numpy(fg)
