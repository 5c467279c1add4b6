"""Writes tests/golden/image_prep.npz: the test pipelines' pixel transforms, restated with cv2 and
numpy the way mmcv runs them, at reduced sizes:

    crop   RandomCrop3D's window img[y1:y1+min(ch, H), x1:x1+min(cw, W)]
           (transforms_3d.py:2527-2542) of uint8 images, offsets as the shipped rel_offsets give
    rescale  mmcv.imrescale: rescale_size (s = min(long / max(h, w), short / min(h, w)),
           int(x * s + 0.5)), then cv2.resize(float32 image, INTER_LINEAR)
    normalise  mmcv.imnormalize_ with the float32 mean / std the Normalize transforms store:
           float32 copy, cv2 BGR->RGB if to_rgb, cv2.subtract of float64(mean), cv2.multiply
           by 1 / float64(std)
    pad    mmcv.impad_to_multiple: cv2.copyMakeBorder to the next multiple, constant 0

Cases: a KITTI-like crop whose source is narrower than the crop (padding on both axes), a
KITTI-like crop inside a larger image (no padding), and Waymo-like rescales limited by the long
side, by the short side, and an upscale.  Run with cv2 installed:

    python tests/golden/make_image_prep_golden.py

cv2.resize is run with IPP disabled: IPP's float linear resize (on in most x86 wheels) rounds
its sample coordinates differently and moves outputs by up to ~1e-4 relative; OpenCV's own
resize is what the CUDA kernel restates.
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# Normalize / MultiViewImageNormalize store img_norm_cfg as float32 (transforms_3d.py:2064-2066)
MEAN = np.array([123.675, 116.28, 103.53], dtype=np.float32)
STD = np.array([58.395, 57.12, 57.375], dtype=np.float32)

# name: (mode, views, src (h, w), crop_size (h, w) or img_scale (long, short), to_rgb)
CASES = {
    'kitti_narrow': ('crop', 1, (25, 150), (20, 160), False),
    'kitti_inside': ('crop', 2, (40, 100), (32, 64), False),
    'waymo_long': ('rescale', 1, (75, 120), (78, 52), True),
    'waymo_short': ('rescale', 1, (75, 90), (78, 52), True),
    'waymo_up': ('rescale', 1, (30, 40), (78, 52), True),
}


def imnormalize(img, mean, std, to_rgb):
    img = img.copy().astype(np.float32)
    mean = np.float64(mean.reshape(1, -1))
    stdinv = 1 / np.float64(std.reshape(1, -1))
    if to_rgb:
        cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
    cv2.subtract(img, mean, img)
    cv2.multiply(img, stdinv, img)
    return img


def impad_to_multiple(img, divisor):
    ph = int(np.ceil(img.shape[0] / divisor)) * divisor
    pw = int(np.ceil(img.shape[1] / divisor)) * divisor
    return cv2.copyMakeBorder(img, 0, ph - img.shape[0], 0, pw - img.shape[1],
                              cv2.BORDER_CONSTANT, value=0)


def crop(img, crop_size, rel_offset_h=(1, 1), rel_offset_w=(0.5, 0.5)):
    margin_h = max(img.shape[0] - crop_size[0], 0)
    margin_w = max(img.shape[1] - crop_size[1], 0)
    y1 = np.random.randint(rel_offset_h[0] * margin_h, rel_offset_h[1] * margin_h + 1)
    x1 = np.random.randint(rel_offset_w[0] * margin_w, rel_offset_w[1] * margin_w + 1)
    ch, cw = min(crop_size[0], img.shape[0]), min(crop_size[1], img.shape[1])
    return img[y1:y1 + ch, x1:x1 + cw], (x1, y1)


def imrescale(img, scale):
    h, w = img.shape[:2]
    s = min(max(scale) / max(h, w), min(scale) / min(h, w))
    size = (int(w * float(s) + 0.5), int(h * float(s) + 0.5))
    return cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)


def run(mode, src, size, to_rgb):
    outs, extra = [], None
    for v in src:
        if mode == 'crop':
            v, extra = crop(v, size)
        else:
            v = imrescale(v.astype(np.float32), size)
        outs.append(impad_to_multiple(imnormalize(v, MEAN, STD, to_rgb), 32))
        content = v.shape[:2]
    return np.stack(outs).transpose(0, 3, 1, 2).copy(), content, extra


def main():
    cv2.ipp.setUseIPP(False)   # this script's own process only
    rng = np.random.RandomState(2024)
    arrays = {}
    for name, (mode, n, hw, size, to_rgb) in CASES.items():
        src = rng.randint(0, 256, (n,) + hw + (3,)).astype(np.uint8)
        out, content, offset = run(mode, src, size, to_rgb)
        arrays[name + '_src'] = src
        arrays[name + '_out'] = out
        arrays[name + '_content'] = np.array(content)
        if offset is not None:
            arrays[name + '_offset'] = np.array(offset)
        print(name, src.shape, '->', out.shape, 'content', content, 'crop', offset)
    np.savez_compressed(os.path.join(HERE, 'image_prep.npz'), **arrays)


if __name__ == '__main__':
    main()
