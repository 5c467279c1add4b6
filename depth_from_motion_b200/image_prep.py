"""The pixel half of the shipped test pipelines on the GPU: decoded 8-bit BGR images in, the
detector's ``img`` tensor and ``img_metas`` out, with no mmcv installed.

``prepare_kitti`` restates the KITTI ``test_pipeline`` (configs/dfm/dfm_r34_1x8_kitti-3d-3class
.py:316-338): per frame ``RandomCrop3D`` (crop_size (320, 1280), rel_offset_h (1, 1),
rel_offset_w (0.5, 0.5)), ``Normalize`` (to_rgb=False) and ``Pad`` (size_divisor 32), applied by
``VideoPipeline`` to the current frame and to each reference frame.  ``prepare_waymo`` restates
the Waymo ``test_pipeline`` (configs/dfm/multiview-dfm_r101_dcn_*.py): ``MultiViewImageResize3D``
(img_scale (1248, 832), keep_ratio: mmcv.imrescale with cv2's float INTER_LINEAR),
``MultiViewImageNormalize`` (to_rgb=True) and ``MultiViewImagePad`` (size_divisor 32).  Both then
stack the views like ``DefaultFormatBundle3D`` (formating.py:43-47), so every view must have the
same size.  The pixels go through one ``dfm_image_prep`` launch; the metadata comes from
``pipeline_meta``.
"""
import ctypes

import numpy as np
import torch

from . import capi, pipeline_meta

IMG_NORM_MEAN = (123.675, 116.28, 103.53)
IMG_NORM_STD = (58.395, 57.12, 57.375)


def _padded(n, divisor):
    return int(np.ceil(n / divisor)) * divisor


def _to_device_views(views, device):
    """Stacks uint8 HWC views into one [N, H, W, 3] CUDA tensor.  numpy or CPU arrays are copied
    through pinned memory; shapes are checked before anything is copied or launched."""
    views = list(views)
    if not views:
        raise ValueError('no images')
    shapes = set()
    for v in views:
        if v.dtype not in (np.uint8, torch.uint8):
            raise ValueError(f'images must be uint8, got {v.dtype}')
        if v.ndim != 3 or v.shape[2] != 3:
            raise ValueError(f'images must be H x W x 3 (BGR), got {tuple(v.shape)}')
        shapes.add(tuple(v.shape))
    if len(shapes) != 1:
        raise ValueError(f'all views must share one size to be stacked, got {sorted(shapes)}')
    if all(isinstance(v, torch.Tensor) and v.is_cuda for v in views):
        return torch.stack([v.to(device) for v in views]).contiguous()
    if any(isinstance(v, torch.Tensor) and v.is_cuda for v in views):
        raise ValueError('mix of CUDA and host images')
    host = torch.empty((len(views),) + shapes.pop(), dtype=torch.uint8, pin_memory=True)
    for i, v in enumerate(views):
        host[i].copy_(torch.as_tensor(np.asarray(v)) if not isinstance(v, torch.Tensor) else v)
    return host.to(device, non_blocking=True)


def image_prep(src, mode, out_hw, crop_xy=(0, 0), size_divisor=32, mean=IMG_NORM_MEAN,
               std=IMG_NORM_STD, to_rgb=False):
    """``dfm_image_prep`` on a CUDA uint8 [N, H, W, 3] tensor -> fp32 [N, 3, Hp, Wp].  ``mean`` and
    ``std`` are the config's ``img_norm_cfg`` values; they are rounded to fp32 first, as
    ``Normalize`` / ``MultiViewImageNormalize`` store them (transforms_3d.py:2064-2066) before
    mmcv.imnormalize widens them back to fp64."""
    n, h, w, _ = src.shape
    desc = capi.ImagePrepDesc()
    desc.mode = capi.DFM_IMAGE_PREP_CROP if mode == 'crop' else capi.DFM_IMAGE_PREP_RESCALE
    desc.num_views, desc.src_h, desc.src_w = n, h, w
    desc.crop_x, desc.crop_y = int(crop_xy[0]), int(crop_xy[1])
    desc.out_h, desc.out_w = int(out_hw[0]), int(out_hw[1])
    desc.pad_divisor, desc.to_rgb = int(size_divisor), int(bool(to_rgb))
    desc.mean[:] = [float(m) for m in np.asarray(mean, dtype=np.float32)]
    desc.std[:] = [float(s) for s in np.asarray(std, dtype=np.float32)]
    out = torch.empty((n, 3, _padded(out_hw[0], size_divisor), _padded(out_hw[1], size_divisor)),
                      device=src.device, dtype=torch.float32)
    with torch.cuda.device(src.device):
        capi.check(capi.lib().dfm_image_prep(
            ctypes.byref(desc), ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(out.data_ptr()),
            ctypes.c_void_p(torch.cuda.current_stream(src.device).cuda_stream)),
            'dfm_image_prep')
    return out


def prepare_kitti(cur, prevs, cam2img, cur2prevs, device='cuda', crop_size=(320, 1280),
                  rel_offset_h=(1, 1), rel_offset_w=(0.5, 0.5), size_divisor=32,
                  mean=IMG_NORM_MEAN, std=IMG_NORM_STD, to_rgb=False):
    """One KITTI sample: ``cur`` and the reference frames ``prevs`` (uint8 H x W x 3 BGR, numpy,
    CPU or CUDA tensors, one size), the current camera's ``cam2img`` and ``cur2prevs``
    ([N_ref, 4, 4], ``pipeline_meta.video_meta``) -> ``(img [1, 1 + N_ref, 3, Hp, Wp],
    [img_meta])`` for ``DfM.simple_test``."""
    views = [cur] + list(prevs)
    if len(views) < 2:
        raise ValueError('DfM needs the current frame and at least one reference frame')
    h, w = views[0].shape[:2]
    # the offsets are drawn per frame; with the shipped fixed rel_offsets they are equal
    x1, y1 = pipeline_meta.random_crop_offsets((h, w), crop_size, rel_offset_h, rel_offset_w)
    ch, cw = min(crop_size[0], h), min(crop_size[1], w)
    src = _to_device_views(views, device)
    img = image_prep(src, 'crop', (ch, cw), (x1, y1), size_divisor, mean, std, to_rgb)
    cropped, crop_offset = pipeline_meta.crop3d_meta(cam2img, x1, y1)
    pad_shape = (img.shape[2], img.shape[3], 3)
    meta = pipeline_meta.backbone_img_meta(cam2img, cur2prevs, (h, w, 3), pad_shape,
                                           crop_offset=crop_offset)
    meta.update(cam2img=cropped.tolist(), img_shape=(ch, cw, 3))
    return img[None], [meta]


def prepare_waymo(views, lidar2img, num_ref_frames=0, device='cuda', img_scale=(1248, 832),
                  size_divisor=32, mean=IMG_NORM_MEAN, std=IMG_NORM_STD, to_rgb=True):
    """One Waymo sample: ``views`` (uint8 H x W x 3 BGR, current frame's cameras first, then
    each reference frame's, all one size) and their ``lidar2img`` ([N, 4, 4], before resizing)
    -> ``(img [1, N, 3, Hp, Wp], [img_meta])`` for ``MultiViewDfM.simple_test``."""
    views = list(views)
    n = len(views)
    if n % (num_ref_frames + 1):
        raise ValueError(f'{n} views do not split into {num_ref_frames + 1} frames')
    lidar2img = np.asarray(lidar2img, dtype=np.float64)
    if lidar2img.shape != (n, 4, 4):
        raise ValueError(f'lidar2img must be [{n}, 4, 4], got {lidar2img.shape}')
    h, w = views[0].shape[:2]
    (nh, nw), scale_factor = pipeline_meta.rescale_meta((h, w), img_scale)
    src = _to_device_views(views, device)
    img = image_prep(src, 'rescale', (nh, nw), (0, 0), size_divisor, mean, std, to_rgb)
    meta = dict(
        ori_lidar2img=lidar2img,
        scale_factor=scale_factor,
        ori_shape=[(h, w, 3)] * n,
        img_shape=[(nh, nw, 3)] * n,
        pad_shape=[(img.shape[2], img.shape[3], 3)] * n,
        num_views=n // (num_ref_frames + 1),
        num_ref_frames=num_ref_frames)
    return img[None], [meta]
