"""dfm_image_prep, the GPU pixel half of the shipped test pipelines (image_prep.py).

CPU: ``prep_reference`` below, a torch restatement of the pipelines' pixel transforms (crop,
cv2's float INTER_LINEAR resize, mmcv.imnormalize, impad_to_multiple), equals the cv2 / numpy
golden written by tests/golden/make_image_prep_golden.py bit for bit, and equals cv2.resize at
the Waymo size (1920 x 1280 -> 1248 x 832) where cv2 is installed.  It is what the GPU tests
compare against at full size, where cv2 need not exist.

GPU: the kernel against the golden and against ``prep_reference`` at the shipped sizes (KITTI
375 x 1242 pair, Waymo 5 and 10 views of 1280 x 1920), with pad cells exactly 0; the metadata
``prepare_kitti`` / ``prepare_waymo`` hand the detectors; malformed input is refused before any
launch.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi, image_prep, pipeline_meta

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
MEAN, STD = image_prep.IMG_NORM_MEAN, image_prep.IMG_NORM_STD
# name: (mode, crop_size or img_scale, to_rgb), as in make_image_prep_golden.CASES
CASES = {'kitti_narrow': ('crop', (20, 160), False), 'kitti_inside': ('crop', (32, 64), False),
         'waymo_long': ('rescale', (78, 52), True), 'waymo_short': ('rescale', (78, 52), True),
         'waymo_up': ('rescale', (78, 52), True)}


# ---------------------------------------------------------------------------------------------
# torch restatement
# ---------------------------------------------------------------------------------------------
def _cv_linear(n_out, n_in, clamp):
    """cv2 resizeGeneric_ INTER_LINEAR coefficients: f = float((d + 0.5) * scale - 0.5) with
    scale = 1 / (double(n_out) / n_in), s = floor(f), w = f - s.  Columns (clamp=True) pin both
    ends to the edge pixel with weight 0; rows keep the weight and clip the two indices."""
    scale = 1.0 / (n_out / n_in)
    f = ((torch.arange(n_out, dtype=torch.float64) + 0.5) * scale - 0.5).to(torch.float32)
    s = torch.floor(f)
    w = f - s
    s = s.long()
    if clamp:
        edge = (s < 0) | (s >= n_in - 1)
        s = torch.where(s < 0, 0, torch.where(s >= n_in - 1, n_in - 1, s))
        w = torch.where(edge, torch.zeros_like(w), w)
    return s.clamp(0, n_in - 1), (s + 1).clamp(0, n_in - 1), w


def cv_resize_linear(img, out_w, out_h):
    """cv2.resize(float32 HWC image, (out_w, out_h), INTER_LINEAR) without IPP: a horizontal
    pass per source row, then the vertical blend, each product and sum rounded to fp32."""
    img = torch.as_tensor(img).float()
    h, w = img.shape[:2]
    x0, x1, ax = _cv_linear(out_w, w, True)
    y0, y1, by = _cv_linear(out_h, h, False)
    ax, a0 = ax[None, :, None], (1 - ax)[None, :, None]
    rows = [img[y][:, x0] * a0 + img[y][:, x1] * ax for y in (y0, y1)]
    return rows[0] * (1 - by)[:, None, None] + rows[1] * by[:, None, None]


def prep_reference(src, mode, size, to_rgb, divisor=32):
    """[N, H, W, 3] uint8 -> [N, 3, Hp, Wp] fp32 as the test pipelines compute it."""
    src = torch.as_tensor(src)
    n, h, w, _ = src.shape
    if mode == 'crop':
        x1, y1 = pipeline_meta.random_crop_offsets((h, w), size, (1, 1), (0.5, 0.5))
        img = src[:, y1:y1 + min(size[0], h), x1:x1 + min(size[1], w)].float()
    else:
        (nh, nw), _ = pipeline_meta.rescale_meta((h, w), size)
        img = torch.stack([cv_resize_linear(v, nw, nh) for v in src])
    if to_rgb:
        img = img.flip(-1)
    # the Normalize transforms store mean / std as float32 (transforms_3d.py:2064-2066);
    # cv2.subtract of the widened scalar runs in fp32, cv2.multiply in fp64 with one rounding
    mean = torch.tensor(MEAN, dtype=torch.float32)
    stdinv = 1 / torch.tensor(STD, dtype=torch.float32).double()
    img = ((img - mean).double() * stdinv).float()
    ch, cw = img.shape[1:3]
    out = torch.zeros((n, 3, -(-ch // divisor) * divisor, -(-cw // divisor) * divisor))
    out[:, :, :ch, :cw] = img.permute(0, 3, 1, 2)
    return out, (ch, cw)


def _golden(name):
    g = np.load(os.path.join(GOLDEN, 'image_prep.npz'))
    return g[name + '_src'], torch.from_numpy(g[name + '_out']), tuple(g[name + '_content'])


def ulps(a, b):
    """Largest distance in fp32 units in the last place between two tensors."""
    ia = a.contiguous().view(torch.int32).long()
    ib = b.contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = torch.where(ib < 0, -(ib & 0x7fffffff), ib)
    return int((ia - ib).abs().max())


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(CASES))
def test_reference_matches_golden(name):
    src, gold, content = _golden(name)
    mode, size, to_rgb = CASES[name]
    got, hw = prep_reference(src, mode, size, to_rgb)
    assert hw == content
    assert torch.equal(got, gold)


def test_reference_resize_matches_cv2_at_waymo_size():
    cv2 = pytest.importorskip('cv2')
    img = np.random.RandomState(5).randint(0, 256, (1280, 1920, 3)).astype(np.float32)
    use_ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)     # OpenCV's own resize: see make_image_prep_golden.py
    try:
        ref = cv2.resize(img, (1248, 832), interpolation=cv2.INTER_LINEAR)
    finally:
        cv2.ipp.setUseIPP(use_ipp)
    assert torch.equal(cv_resize_linear(img, 1248, 832), torch.from_numpy(ref))


def test_normalise_uses_the_float32_cfg_like_the_transforms():
    """mmcv.imnormalize as Normalize / MultiViewImageNormalize call it (mean / std stored as
    np.float32, transforms_3d.py:2064-2066), over every uint8 value of every channel; the
    config's float64 std would differ in the last place for some of them."""
    cv2 = pytest.importorskip('cv2')
    x = np.arange(256, dtype=np.float32).reshape(1, 256, 1).repeat(3, 2)
    mean, std = np.array(MEAN, dtype=np.float32), np.array(STD, dtype=np.float32)
    ref = x.copy()
    cv2.subtract(ref, np.float64(mean.reshape(1, -1)), ref)
    cv2.multiply(ref, 1 / np.float64(std.reshape(1, -1)), ref)
    src = torch.from_numpy(x.astype(np.uint8)[None])
    got, _ = prep_reference(src, 'crop', (1, 256), False, divisor=1)
    assert torch.equal(got[0].permute(1, 2, 0), torch.from_numpy(ref))
    widened = ((torch.from_numpy(x) - torch.tensor(MEAN).float()).double() *
               (1 / torch.tensor(STD, dtype=torch.float64))).float()
    assert not torch.equal(widened, torch.from_numpy(ref))


def test_rescale_meta_of_the_shipped_sizes():
    (h, w), sf = pipeline_meta.rescale_meta((1280, 1920), (1248, 832))
    assert (h, w) == (832, 1248)
    assert sf.dtype == np.float32 and np.array_equal(sf, np.float32([0.65] * 4))
    (h, w), sf = pipeline_meta.rescale_meta((886, 1920), (1248, 832))
    assert (h, w) == (576, 1248)
    assert np.array_equal(sf, np.float32([1248 / 1920, 576 / 886] * 2))


def test_malformed_input_is_refused_before_any_launch():
    a = np.zeros((40, 60, 3), np.uint8)
    with pytest.raises(ValueError, match='one size'):
        image_prep.prepare_waymo([a, np.zeros((40, 62, 3), np.uint8)], np.stack([np.eye(4)] * 2))
    with pytest.raises(ValueError, match='one size'):
        image_prep.prepare_kitti(a, [np.zeros((41, 60, 3), np.uint8)], np.eye(4), np.eye(4)[None])
    with pytest.raises(ValueError, match='uint8'):
        image_prep.prepare_waymo([a.astype(np.float32)], np.eye(4)[None])
    with pytest.raises(ValueError, match='H x W x 3'):
        image_prep.prepare_waymo([np.zeros((40, 60), np.uint8)], np.eye(4)[None])
    with pytest.raises(ValueError, match='lidar2img'):
        image_prep.prepare_waymo([a, a], np.eye(4)[None])
    with pytest.raises(ValueError, match='frames'):
        image_prep.prepare_waymo([a] * 5, np.stack([np.eye(4)] * 5), num_ref_frames=1)
    with pytest.raises(ValueError, match='reference frame'):
        image_prep.prepare_kitti(a, [], np.eye(4), np.eye(4)[None])


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _kernel(src, name_or_mode, size, to_rgb):
    mode = name_or_mode
    n, h, w, _ = src.shape
    if mode == 'crop':
        x1, y1 = pipeline_meta.random_crop_offsets((h, w), size, (1, 1), (0.5, 0.5))
        out_hw = (min(size[0], h), min(size[1], w))
    else:
        x1 = y1 = 0
        out_hw, _ = pipeline_meta.rescale_meta((h, w), size)
    out = image_prep.image_prep(src, mode, out_hw, (x1, y1), 32, MEAN, STD, to_rgb)
    capi.sync_check()
    return out.cpu(), out_hw


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_kernel_matches_golden(name):
    src, gold, content = _golden(name)
    mode, size, to_rgb = CASES[name]
    got, hw = _kernel(torch.from_numpy(src).cuda(), mode, size, to_rgb)
    assert tuple(hw) == content and got.shape == gold.shape
    u = ulps(got, gold)
    print(name, 'max fp32 ulps from the golden', u)
    if mode == 'crop':
        assert torch.equal(got, gold)
    else:
        assert u <= 4


@pytest.mark.gpu
@pytest.mark.parametrize('mode,n,hw,size,to_rgb', [
    ('crop', 2, (375, 1242), (320, 1280), False),
    ('rescale', 5, (1280, 1920), (1248, 832), True),
    ('rescale', 10, (1280, 1920), (1248, 832), True)])
def test_kernel_matches_reference_at_full_size(mode, n, hw, size, to_rgb):
    src = torch.from_numpy(np.random.RandomState(n).randint(0, 256, (n,) + hw + (3,),
                                                            dtype=np.uint8))
    ref, (ch, cw) = prep_reference(src, mode, size, to_rgb)
    got, out_hw = _kernel(src.cuda(), mode, size, to_rgb)
    assert got.shape == ref.shape
    assert tuple(out_hw) == (ch, cw)
    u = ulps(got, ref)
    print(mode, n, hw, 'output', tuple(got.shape), 'max fp32 ulps from the reference', u)
    assert u <= (0 if mode == 'crop' else 4)
    assert not got[:, :, ch:].any() and not got[:, :, :, cw:].any()


@pytest.mark.gpu
def test_prepare_kitti_and_waymo_shapes_and_metas():
    rng = np.random.RandomState(3)
    cur, prev = (rng.randint(0, 256, (375, 1242, 3), dtype=np.uint8) for _ in range(2))
    k = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.2], [0, 0, 1, 0.003],
                  [0, 0, 0, 1]])
    c2p = np.eye(4)[None]
    c2p[0, 2, 3] = -0.8
    img, metas = image_prep.prepare_kitti(cur, [prev], k, c2p)
    assert img.shape == (1, 2, 3, 320, 1248) and img.is_cuda
    m = metas[0]
    assert m['crop_offset'] == [0, 55] and m['pad_shape'] == (320, 1248, 3)
    assert m['img_shape'] == (320, 1242, 3) and m['ori_shape'] == (375, 1242, 3)
    assert np.allclose(np.asarray(m['cam2img'])[1, 2], 172.9 - 55)
    assert m['cur2prevs'].dtype == torch.float32 and m['cur2prevs'].shape == (1, 4, 4)
    # CUDA input gives the same tensor as host input
    img2, _ = image_prep.prepare_kitti(torch.from_numpy(cur).cuda(),
                                       [torch.from_numpy(prev).cuda()], k, c2p)
    assert torch.equal(img, img2)
    views = [rng.randint(0, 256, (1280, 1920, 3), dtype=np.uint8) for _ in range(10)]
    l2i = np.stack([np.eye(4)] * 10)
    img, metas = image_prep.prepare_waymo(views, l2i, num_ref_frames=1)
    assert img.shape == (1, 10, 3, 832, 1248)
    m = metas[0]
    assert (m['num_views'], m['num_ref_frames']) == (5, 1)
    assert m['img_shape'] == [(832, 1248, 3)] * 10 and m['pad_shape'] == [(832, 1248, 3)] * 10
    assert np.array_equal(m['scale_factor'], np.float32([0.65] * 4))
    capi.sync_check()


@pytest.mark.gpu
def test_c_abi_refuses_what_it_cannot_serve():
    src = torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device='cuda')
    out = torch.empty((1, 3, 32, 32), device='cuda')
    L = capi.lib()

    def call(**kw):
        d = capi.ImagePrepDesc()
        base = dict(mode=0, num_views=1, src_h=8, src_w=8, out_h=8, out_w=8, pad_divisor=32)
        for key, v in {**base, **kw}.items():
            setattr(d, key, v)
        d.mean[:] = list(MEAN)
        d.std[:] = list(kw.pop('std', STD))
        return L.dfm_image_prep(ctypes.byref(d), ctypes.c_void_p(src.data_ptr()),
                                ctypes.c_void_p(out.data_ptr()), None)
    assert call() == capi.DFM_OK
    invalid = 1
    assert call(crop_x=1) == invalid                       # window leaves the image
    assert call(out_h=0) == invalid
    assert call(mode=2) == invalid
    assert call(pad_divisor=0) == invalid
    assert call(mode=1, out_h=4, out_w=4) == invalid       # exact 2x: cv2 runs INTER_AREA
    assert call(std=(0.0, 1.0, 1.0)) == invalid
    capi.sync_check()
