"""Input-side metadata the DfM hot path reads (SURVEY.md section 8(f) row 4): what the
reference's data pipeline puts into ``img_metas`` for ``DfMBackbone.forward``
(dfm_backbone.py:150-172) and for MultiViewDfM's lifting.  Host-side NumPy only -- no images
are touched here; the pixel half of the test pipelines (crop / resize / normalise / pad) runs
on the GPU in ``image_prep.py``, which builds its metadata from these functions.  Restated
from:

    VideoPipeline.__call__     mmdet3d/datasets/pipelines/loading.py:416-545
        reference-frame selection (:434-444), cam2global (:451-468, :495-513),
        cur2prev = inv(prev_cam2global) @ cur_cam2global (:530-537), stacked (:541)
    RandomCrop3D._crop_data    mmdet3d/datasets/pipelines/transforms_3d.py:2530-2537 (offsets),
        :2583-2594 (intrinsics after the crop, ``crop_offset``)
    DfM.extract_feat           mmdet3d/models/detectors/dfm.py:288-293 (cur2prevs -> tensor)
    MultiViewImageResize3D._resize_img  transforms_3d.py:2409-2434 (mmcv.imrescale size,
        ``scale_factor``)
"""
import numpy as np


def select_ref_frames(num_sweeps, num_ref_imgs=-1, random=True, rng=None):
    """Indices of the reference (previous) frames, loading.py:434-444: ``num_ref_imgs`` random
    sweeps (with replacement only if there are fewer sweeps than requested) in training, the
    LAST ``num_ref_imgs`` sweeps in test mode (``random=False``); none if ``num_ref_imgs <= 0``."""
    if num_ref_imgs > 0 and num_sweeps:
        ids = np.arange(num_sweeps)
        if random:
            rng = rng or np.random
            replace = num_ref_imgs > len(ids)
            return rng.choice(ids, num_ref_imgs, replace=replace)
        return ids[-num_ref_imgs:]
    return np.arange(0)


def quaternion_matrix(q):
    """4x4 homogeneous rotation of a unit quaternion (w, x, y, z):
    pyquaternion's ``Quaternion(q).transformation_matrix`` used at loading.py:452-468."""
    w, x, y, z = (float(v) for v in q)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    m = np.eye(4)
    m[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    return m


def cam2global_of(info, nuscenes_keys=('cam2ego_rotation', 'cam2ego_translation')):
    """Camera-to-global pose of a frame record: KITTI / Waymo infos carry ``cam2global``
    (loading.py:468, :513); nuScenes-style records compose cam2ego and ego2global
    (:451-466 for the key frame, :495-511 for a sweep, whose keys are ``sensor2ego_*``)."""
    if 'cam2global' in info:
        return np.asarray(info['cam2global'])
    rot_k, tr_k = nuscenes_keys
    cam2ego = quaternion_matrix(info[rot_k])
    cam2ego[0:3, 3] += np.array(info[tr_k]).T
    ego2global = quaternion_matrix(info['ego2global_rotation'])
    ego2global[0:3, 3] += np.array(info['ego2global_translation']).T
    return np.dot(ego2global, cam2ego).astype(np.float32)


def _pad4(m):
    p = np.eye(4)
    m = np.asarray(m)
    p[:m.shape[0], :m.shape[1]] = m
    return p


def cur2prevs(cur_cam2global, prev_cam2globals):
    """[N_ref, 4, 4] float64: ``inv(pad(prev)) @ pad(cur)`` per reference frame
    (loading.py:476-479, 530-537, 541)."""
    cur = _pad4(cur_cam2global)
    return np.stack([np.linalg.inv(_pad4(p)).dot(cur) for p in prev_cam2globals], axis=0)


def video_meta(img_info, num_ref_imgs=-1, random=True, rng=None):
    """The geometric part of VideoPipeline.__call__ for one sample's ``img_info`` (with
    ``sweeps``): selected sweep indices, their file names and ``cur2prevs``."""
    sweeps = img_info.get('sweeps', [])
    ids = select_ref_frames(len(sweeps), num_ref_imgs, random, rng)
    cur = cam2global_of(img_info)
    prevs = [cam2global_of(sweeps[i], ('sensor2ego_rotation', 'sensor2ego_translation'))
             for i in ids.tolist()]
    out = dict(ref_ids=ids, ref_filenames=[sweeps[i].get('data_path') for i in ids.tolist()],
               cam2global=cur)
    if prevs:
        out['cur2prevs'] = cur2prevs(cur, prevs)
    return out


def random_crop_offsets(img_shape, crop_size, rel_offset_h=(0., 1.), rel_offset_w=(0., 1.),
                        rng=None):
    """(crop_x1, crop_y1) like RandomCrop3D._crop_data (transforms_3d.py:2530-2537): h first,
    then w, ``randint(lo * margin, hi * margin + 1)``."""
    rng = rng or np.random
    margin_h = max(img_shape[0] - crop_size[0], 0)
    margin_w = max(img_shape[1] - crop_size[1], 0)
    offset_h = rng.randint(rel_offset_h[0] * margin_h, rel_offset_h[1] * margin_h + 1)
    offset_w = rng.randint(rel_offset_w[0] * margin_w, rel_offset_w[1] * margin_w + 1)
    return int(offset_w), int(offset_h)


def crop3d_meta(cam2img, crop_x1, crop_y1):
    """Intrinsics after a crop at (crop_x1, crop_y1) and the ``crop_offset`` meta key
    (transforms_3d.py:2583-2592): the principal point of K moves, P = K' (K^-1 P)."""
    cam2img = np.array(cam2img, dtype=np.float64, copy=True)
    K = cam2img[:3, :3].copy()
    T = np.matmul(np.linalg.inv(K), cam2img[:3])
    K[0, 2] -= crop_x1
    K[1, 2] -= crop_y1
    off = np.matmul(K, T)
    cam2img[:off.shape[0], :off.shape[1]] = off
    return cam2img, [crop_x1, crop_y1]


def rescale_meta(img_hw, img_scale):
    """Size and ``scale_factor`` of a keep-ratio resize (MultiViewImageResize3D, keep_ratio=True):
    mmcv ``rescale_size`` takes ``s = min(long / max(h, w), short / min(h, w))`` for the
    (long, short) ``img_scale`` and the new size ``int(x * s + 0.5)``; the recorded factor is the
    one actually applied per axis, ``[w_scale, h_scale, w_scale, h_scale]`` in fp32
    (transforms_3d.py:2418-2434).  Returns ``((new_h, new_w), scale_factor)``."""
    h, w = img_hw
    s = min(max(img_scale) / max(h, w), min(img_scale) / min(h, w))
    new_w, new_h = int(w * float(s) + 0.5), int(h * float(s) + 0.5)
    w_scale, h_scale = new_w / w, new_h / h
    return (new_h, new_w), np.array([w_scale, h_scale, w_scale, h_scale], dtype=np.float32)


def backbone_img_meta(ori_cam2img, cur2prevs_np, ori_shape, pad_shape, crop_offset=(0, 0),
                      scale_factor=1.0, flip=False):
    """The ``img_metas[i]`` entry DfMBackbone.forward reads (dfm_backbone.py:150-172), with
    ``cur2prevs`` already converted like DfM.extract_feat does (detectors/dfm.py:288-293)."""
    import torch
    return dict(ori_cam2img=np.asarray(ori_cam2img, dtype=np.float32).tolist(),
                cur2prevs=torch.as_tensor(np.asarray(cur2prevs_np), dtype=torch.float32),
                ori_shape=tuple(ori_shape), pad_shape=tuple(pad_shape), img_shape=tuple(pad_shape),
                crop_offset=list(crop_offset), flip=bool(flip),
                scale_factor=[scale_factor] * 4)
