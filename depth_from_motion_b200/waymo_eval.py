"""Building blocks of Waymo's camera-only LET-3D-AP (``WaymoDataset.evaluate(metric='waymo')``
with ``cam_sync=True``, which runs Waymo's ``compute_detection_let_metrics_main``).

- ``read_objects`` / ``write_objects``: a pure-Python protobuf wire codec for the fields of
  ``metrics_pb2.Objects`` the metric reads, so a ``cam_gt.bin`` can be read and a
  submission ``.bin`` written without TensorFlow or the Waymo package.  The writer emits the
  bytes protobuf's serialiser emits for the same set fields.
- ``let_iou``: the metric's pair stage on the device (``csrc/waymo_eval_kernels.cuh``): the
  longitudinal alignment, the fp64 3-D rotated IoU, the longitudinal affinity and the
  heading accuracy of every (prediction, GT) pair.

It also holds WaymoDataset's second metric, ``evaluate(metric='kitti')`` for load_mode
'lidar_frame' (both MultiViewDfM configs): ``convert_valid_bboxes`` / ``bbox2result_kitti`` run
for the whole set in one launch of ``dfm_waymo_kitti_convert``, and ``kitti_eval`` scores the
result in column form, in parts of frames that fit its overlap limit.
"""
import ctypes
import struct

import numpy as np

from . import capi

# ---------------------------------------------------------------------------------------
# protobuf wire codec of Objects (waymo_open_dataset/protos/metrics.proto, label.proto)
# ---------------------------------------------------------------------------------------
# presence bits of the optional fields of one object (proto2: a field is written iff set)
HAS_BOX, HAS_TYPE, HAS_ID, HAS_DIFFICULTY, HAS_NUM_POINTS, HAS_CAMERA, HAS_SYNCED_BOX, \
    HAS_SCORE, HAS_LABEL = (1 << i for i in range(9))

# Label.Box field numbers in serialisation order and their column in the [n, 7] box arrays
# (columns: center_x, center_y, center_z, length, width, height, heading)
_BOX_FIELDS = ((1, 0), (2, 1), (3, 2), (4, 4), (5, 3), (6, 5), (7, 6))
_BOX_COL = {f: c for f, c in _BOX_FIELDS}


def _varint(n):
    if n < 0:
        n += 1 << 64
    out = bytearray()
    while True:
        b = n & 0x7f
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _read_varint(buf, i):
    r = s = 0
    while True:
        if i >= len(buf):
            raise ValueError('truncated varint')
        c = buf[i]
        i += 1
        r |= (c & 0x7f) << s
        s += 7
        if c < 0x80:
            return r, i


def _fields(buf):
    """Yields (field number, wire type, value) of one message; a length-delimited value is
    a memoryview, fixed64 / fixed32 values are their raw bytes."""
    i, n = 0, len(buf)
    while i < n:
        tag, i = _read_varint(buf, i)
        f, wt = tag >> 3, tag & 7
        if wt == 0:
            v, i = _read_varint(buf, i)
        elif wt == 1:
            v, i = buf[i:i + 8], i + 8
        elif wt == 2:
            ln, i = _read_varint(buf, i)
            v, i = buf[i:i + ln], i + ln
        elif wt == 5:
            v, i = buf[i:i + 4], i + 4
        else:
            raise ValueError(f'unsupported wire type {wt}')
        if i > n:
            raise ValueError('truncated message')
        yield f, wt, v


def _signed64(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= 1 << 63 else v


def _parse_box(buf, row):
    for f, wt, v in _fields(buf):
        if f in _BOX_COL and wt == 1:
            row[_BOX_COL[f]] = struct.unpack('<d', v)[0]


def _new_frame(context_name, timestamp):
    return {'context_name': context_name, 'frame_timestamp_micros': timestamp,
            'box': [], 'type': [], 'score': [], 'id': [], 'detection_difficulty_level': [],
            'num_lidar_points_in_box': [], 'most_visible_camera_name': [],
            'camera_synced_box': [], 'has': []}


def _finish_frame(fr):
    n = len(fr['type'])
    fr['box'] = np.asarray(fr['box'], np.float64).reshape(n, 7)
    fr['camera_synced_box'] = np.asarray(fr['camera_synced_box'], np.float64).reshape(n, 7)
    fr['type'] = np.asarray(fr['type'], np.int32)
    fr['score'] = np.asarray(fr['score'], np.float32)
    fr['detection_difficulty_level'] = np.asarray(fr['detection_difficulty_level'], np.int32)
    fr['num_lidar_points_in_box'] = np.asarray(fr['num_lidar_points_in_box'], np.int32)
    fr['has'] = np.asarray(fr['has'], np.int32)
    return fr


def read_objects(path_or_bytes):
    """Parses a serialised ``Objects`` into frames, in the order of their first object.

    A frame is a dict with ``context_name``, ``frame_timestamp_micros`` and, per object,
    ``box`` / ``camera_synced_box`` [n, 7] fp64 (center x, y, z, length, width, height,
    heading), ``type`` int32, ``score`` float32 (1 when unset, the proto default), ``id``,
    ``detection_difficulty_level`` and ``num_lidar_points_in_box`` int32,
    ``most_visible_camera_name`` and ``has``, the HAS_* bits of the fields that were set.
    Unset numbers read as 0, unset strings as ''.  Fields the metric does not read are
    skipped."""
    if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
        buf = memoryview(bytes(path_or_bytes))
    else:
        with open(path_or_bytes, 'rb') as f:
            buf = memoryview(f.read())
    frames = {}
    for f, wt, obj in _fields(buf):
        if f != 1 or wt != 2:
            continue
        label, score, ctx, ts, has = None, 1.0, '', 0, 0
        for g, wt2, v in _fields(obj):
            if g == 1 and wt2 == 2:
                label, has = v, has | HAS_LABEL
            elif g == 2 and wt2 == 5:
                score, has = struct.unpack('<f', v)[0], has | HAS_SCORE
            elif g == 4 and wt2 == 2:
                ctx = bytes(v).decode('utf-8')
            elif g == 5 and wt2 == 0:
                ts = _signed64(v)
        key = (ctx, ts)
        fr = frames.get(key)
        if fr is None:
            fr = frames[key] = _new_frame(ctx, ts)
        box, sbox = [0.0] * 7, [0.0] * 7
        typ = diff = npts = 0
        oid = cam = ''
        if label is not None:
            for g, wt2, v in _fields(label):
                if g == 1 and wt2 == 2:
                    _parse_box(v, box)
                    has |= HAS_BOX
                elif g == 3 and wt2 == 0:
                    typ, has = _signed64(v), has | HAS_TYPE
                elif g == 4 and wt2 == 2:
                    oid, has = bytes(v).decode('utf-8'), has | HAS_ID
                elif g == 5 and wt2 == 0:
                    diff, has = _signed64(v), has | HAS_DIFFICULTY
                elif g == 7 and wt2 == 0:
                    npts, has = _signed64(v), has | HAS_NUM_POINTS
                elif g == 11 and wt2 == 2:
                    cam, has = bytes(v).decode('utf-8'), has | HAS_CAMERA
                elif g == 12 and wt2 == 2:
                    _parse_box(v, sbox)
                    has |= HAS_SYNCED_BOX
        fr['box'].append(box)
        fr['camera_synced_box'].append(sbox)
        fr['type'].append(typ)
        fr['score'].append(score)
        fr['id'].append(oid)
        fr['detection_difficulty_level'].append(diff)
        fr['num_lidar_points_in_box'].append(npts)
        fr['most_visible_camera_name'].append(cam)
        fr['has'].append(has)
    return [_finish_frame(fr) for fr in frames.values()]


def _len_field(f, payload):
    return _varint(f << 3 | 2) + _varint(len(payload)) + payload


def _box_bytes(row):
    return b''.join(_varint(f << 3 | 1) + struct.pack('<d', float(row[c]))
                    for f, c in _BOX_FIELDS)


def _object_bytes(fr, i):
    has = int(fr['has'][i]) if 'has' in fr else (
        HAS_LABEL | HAS_BOX | HAS_TYPE | HAS_SCORE)
    lab = b''
    if has & HAS_BOX:
        lab += _len_field(1, _box_bytes(fr['box'][i]))
    if has & HAS_TYPE:
        lab += _varint(3 << 3) + _varint(int(fr['type'][i]))
    if has & HAS_ID:
        lab += _len_field(4, fr['id'][i].encode('utf-8'))
    if has & HAS_DIFFICULTY:
        lab += _varint(5 << 3) + _varint(int(fr['detection_difficulty_level'][i]))
    if has & HAS_NUM_POINTS:
        lab += _varint(7 << 3) + _varint(int(fr['num_lidar_points_in_box'][i]))
    if has & HAS_CAMERA:
        lab += _len_field(11, fr['most_visible_camera_name'][i].encode('utf-8'))
    if has & HAS_SYNCED_BOX:
        lab += _len_field(12, _box_bytes(fr['camera_synced_box'][i]))
    obj = b''
    if has & HAS_LABEL:
        obj += _len_field(1, lab)
    if has & HAS_SCORE:
        obj += _varint(2 << 3 | 5) + struct.pack('<f', float(fr['score'][i]))
    obj += _len_field(4, fr['context_name'].encode('utf-8'))
    obj += _varint(5 << 3) + _varint(int(fr['frame_timestamp_micros']))
    return _len_field(1, obj)


def objects_bytes(frames):
    """The serialised ``Objects`` of ``frames`` (see ``read_objects``), objects in frame
    order.  Without a ``has`` entry a frame's objects carry box, type and score.  A set box
    is written with all seven of its fields."""
    return b''.join(_object_bytes(fr, i) for fr in frames for i in range(len(fr['type'])))


def write_objects(path, frames):
    """Writes ``objects_bytes(frames)`` to ``path`` (a submission or GT ``.bin``)."""
    with open(path, 'wb') as f:
        f.write(objects_bytes(frames))


# ---------------------------------------------------------------------------------------
# LET pair stage on the device
# ---------------------------------------------------------------------------------------
# IoU threshold per type (UNKNOWN, VEHICLE, PEDESTRIAN, SIGN, CYCLIST) as the binary's config
# stores them; it compares float32(LET-IoU) against them
IOU_THRESHOLDS = np.array([0.0, 0.5, 0.3, 0.3, 0.3], np.float32)


def let_iou(pred_boxes, gt_boxes):
    """[n, k, 3] fp64 on the GPU: (LET-IoU, longitudinal affinity, heading accuracy) of every
    (prediction, GT) pair; boxes are [., 7] (center x, y, z, length, width, height, heading)
    in the vehicle frame.  See ``dfm_op_let_iou`` in ``include/dfm_b200.h``."""
    import torch
    pd = torch.as_tensor(pred_boxes, dtype=torch.float64).reshape(-1, 7)
    gt = torch.as_tensor(gt_boxes, dtype=torch.float64).reshape(-1, 7)
    n, k = pd.shape[0], gt.shape[0]
    if n == 0 or k == 0:
        return torch.zeros(n, k, 3, dtype=torch.float64, device='cuda')
    pd = pd.to('cuda').contiguous()
    gt = gt.to('cuda').contiguous()
    out = torch.empty(n, k, 3, dtype=torch.float64, device='cuda')
    capi.check(capi.lib().dfm_op_let_iou(
        ctypes.c_void_p(pd.data_ptr()), ctypes.c_void_p(gt.data_ptr()), n, k,
        ctypes.c_void_p(out.data_ptr()),
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'dfm_op_let_iou')
    return out


def matchable(let_iou_out, gt_types):
    """[n, k] bool: pairs that may match, affinity > 0 and float32(LET-IoU) >= the GT
    type's threshold (the caller keeps only same-type pairs)."""
    thr = IOU_THRESHOLDS[np.asarray(gt_types, np.int64)]
    v = np.asarray(let_iou_out, np.float64)
    return (v[..., 1] > 0.0) & (v[..., 0].astype(np.float32) >= thr[None, :])


# ---------------------------------------------------------------------------------------
# WaymoDataset.evaluate(metric='kitti') for load_mode 'lidar_frame' (both MultiViewDfM
# configs): convert_valid_bboxes / bbox2result_kitti on the device, then kitti_eval
# ---------------------------------------------------------------------------------------
WAYMO_PCD_LIMIT_RANGE = (-85, -85, -5, 85, 85, 5)
# class_names of both MultiViewDfM configs, which set WaymoDataset.CLASSES: label 0 is
# 'Pedestrian'
WAYMO_CLASSES = ('Pedestrian', 'Cyclist', 'Car')
ANNO_KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
             'rotation_y', 'score')
CONVERT_W = 17   # columns of dfm_waymo_kitti_convert's output


def _unwrap(results):
    if len(results) == 0:
        raise ValueError('no results')
    if not isinstance(results[0], dict):
        raise ValueError('2-D-only results (bbox2result_kitti2d) are not supported')
    for r in results:
        missing = [k for k in ('boxes_3d', 'scores_3d', 'labels_3d') if k not in r]
        if missing:
            raise ValueError(f'a result lacks {missing}')
    return results


def _calib_rows(data_infos):
    """[frames][32] float32: R0_rect @ Tr_velo_to_cam as the reference forms it (a float32
    numpy product per frame), then P0; [frames][2] image shapes; [frames] image_idx."""
    calib = np.empty((len(data_infos), 32), np.float32)
    shape = np.empty((len(data_infos), 2), np.int32)
    idx = np.empty(len(data_infos), np.int64)
    for f, info in enumerate(data_infos):
        c = info['calib']
        rt = c['R0_rect'].astype(np.float32) @ c['Tr_velo_to_cam'].astype(np.float32)
        p0 = np.asarray(c['P0'], np.float32)
        if rt.shape != (4, 4) or p0.shape != (4, 4):
            raise ValueError(f'data_infos[{f}]: R0_rect, Tr_velo_to_cam and P0 must be 4 x 4')
        calib[f, :16] = rt.reshape(-1)
        calib[f, 16:] = p0.reshape(-1)
        shape[f] = np.asarray(info['image']['image_shape'])[:2]
        idx[f] = int(info['image']['image_idx'])
    return calib, shape, idx


def convert_set(results, data_infos, pcd_limit_range=WAYMO_PCD_LIMIT_RANGE):
    """``convert_valid_bboxes`` of every frame in one launch of ``dfm_waymo_kitti_convert``.

    Returns per box of the set (frame order): ``off`` [frames + 1], ``keep`` bool, ``out``
    [boxes][17] float32 (see ``include/dfm_b200.h``), ``boxes`` [boxes][7] float32 (the
    input LiDAR boxes), ``scores`` and ``labels`` as numpy, and ``sample_idx`` int64."""
    d = _convert(results, data_infos, pcd_limit_range)
    return dict(off=d['off'], keep=d['keep'].cpu().numpy().astype(bool),
                out=d['out'].cpu().numpy(), boxes=d['boxes'].cpu().numpy(), scores=d['scores'],
                labels=d['labels'], sample_idx=d['sample_idx'].cpu().numpy())


def _convert(results, data_infos, pcd_limit_range):
    """``convert_set`` with keep, out, boxes and sample_idx left on the device."""
    import torch
    results = _unwrap(results)
    if len(results) != len(data_infos):
        raise ValueError(f'{len(results)} results but {len(data_infos)} data_infos')
    if len(pcd_limit_range) != 6:
        raise ValueError('pcd_limit_range must hold 6 values')
    from .kitti_eval import _boxes_tensor
    boxes = [_boxes_tensor(r['boxes_3d']) for r in results]
    scores = [torch.as_tensor(r['scores_3d']).detach().cpu() for r in results]
    labels = [torch.as_tensor(r['labels_3d']).detach().cpu() for r in results]
    n = np.array([len(b) for b in boxes], np.int64)
    if any(len(s) != k or len(l) != k for s, l, k in zip(scores, labels, n)):
        raise ValueError('boxes_3d, scores_3d and labels_3d differ in length')
    off = np.concatenate([[0], np.cumsum(n)])
    K = int(off[-1])
    if K >= 1 << 31:
        raise ValueError(f'{K} boxes, more than the int32 offsets index')
    calib, shape, idx = _calib_rows(data_infos)
    dev = torch.device('cuda')
    keep = torch.empty(K, dtype=torch.uint8, device=dev)
    out = torch.empty(K, CONVERT_W, dtype=torch.float32, device=dev)
    sidx = torch.empty(K, dtype=torch.int64, device=dev)
    t_boxes = torch.cat(boxes).to(dev).contiguous()
    t_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    t_calib = torch.from_numpy(calib).to(dev)
    t_shape = torch.from_numpy(shape).to(dev)
    t_idx = torch.from_numpy(idx).to(dev)
    p = lambda x: ctypes.c_void_p(x.data_ptr()) if x.numel() else None
    lim = (ctypes.c_float * 6)(*[float(v) for v in pcd_limit_range])
    capi.check(capi.lib().dfm_waymo_kitti_convert(
        len(data_infos), K, p(t_boxes), p(t_off), p(t_calib), p(t_shape), p(t_idx), lim,
        p(keep), p(out), p(sidx), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
        'dfm_waymo_kitti_convert')
    return dict(off=off, keep=keep, out=out, boxes=t_boxes, sample_idx=sidx,
                scores=torch.cat(scores).numpy() if K else np.zeros(0, np.float32),
                labels=torch.cat(labels).numpy() if K else np.zeros(0, np.int64))


def convert_valid_bboxes(box_dict, info, pcd_limit_range=WAYMO_PCD_LIMIT_RANGE):
    """WaymoDataset.convert_valid_bboxes, load_mode 'lidar_frame', on the device: the 2-D
    box of the P0 projection, the camera and LiDAR boxes, scores and labels of the boxes whose
    centre lies strictly inside ``pcd_limit_range``.  ``boxes_3d`` is a [K, 7] tensor (or a
    box structure with ``.tensor``) in LiDAR coordinates, bottom centre."""
    c = convert_set([box_dict], [info], pcd_limit_range)
    sample_idx = info['image']['image_idx']
    v = c['keep']
    if not v.any():
        return dict(bbox=np.zeros([0, 4]), box3d_camera=np.zeros([0, 7]),
                    box3d_lidar=np.zeros([0, 7]), scores=np.zeros([0]),
                    label_preds=np.zeros([0]), sample_idx=sample_idx)
    o = c['out'][v]
    lidar = c['boxes'][v].copy()
    lidar[:, 6] = o[:, 12]
    return dict(bbox=np.ascontiguousarray(o[:, 13:17]),
                box3d_camera=np.ascontiguousarray(o[:, [5, 6, 7, 8, 9, 10, 11]]),
                box3d_lidar=lidar, scores=c['scores'][v], label_preds=c['labels'][v],
                sample_idx=sample_idx)


def _kept_columns(c, class_names, with_names=True):
    """The anno columns of the kept boxes and their frame offsets.  ``code`` holds the
    evaluator's class code of each box, looked up per class from its label; ``name`` (with
    ``with_names``) the class name."""
    from .kitti_eval import name_codes
    v = c['keep']
    labels = c['labels'][v].astype(np.int64)
    if len(labels) and (labels.min() < 0 or labels.max() >= len(class_names)):
        bad = labels[(labels < 0) | (labels >= len(class_names))][0]
        raise ValueError(f'label {int(bad)} has no class name')
    o = c['out'][v]
    kept_before = np.concatenate([[0], np.cumsum(v, dtype=np.int64)])
    names = np.asarray(list(class_names))
    cols = dict(code=name_codes(names, False)[labels], alpha=o[:, 4], bbox=o[:, 0:4],
                location=o[:, 5:8], dimensions=o[:, 8:11], rotation_y=o[:, 11],
                score=c['scores'][v], sample_idx=c['sample_idx'][v],
                name_len=np.array([len(x) for x in class_names], np.int64)[labels])
    if with_names:
        cols['name'] = names[labels] if len(labels) else np.zeros(0, '<U1')
    return cols, kept_before[np.asarray(c['off'], np.int64)]


def _empty_anno():
    return {'name': np.array([]), 'truncated': np.array([]), 'occluded': np.array([]),
            'alpha': np.array([]), 'bbox': np.zeros([0, 4]), 'dimensions': np.zeros([0, 3]),
            'location': np.zeros([0, 3]), 'rotation_y': np.array([]), 'score': np.array([]),
            'sample_idx': np.array([], dtype=np.int64)}


def _write_submissions(prefix, cols, off, data_infos):
    """``<prefix>/<sample_idx:07d>.txt`` in the benchmark's format for every frame that keeps
    a box, as the reference writes them."""
    import os
    os.makedirs(prefix, exist_ok=True)
    b, loc, dims = cols['bbox'], cols['location'], cols['dimensions']
    for f in np.flatnonzero(np.diff(off) > 0):
        idx = int(data_infos[f]['image']['image_idx'])
        with open(f'{prefix}/{idx:07d}.txt', 'w') as fh:
            for i in range(int(off[f]), int(off[f + 1])):
                print('{} -1 -1 {:.4f} {:.4f} {:.4f} {:.4f} {:.4f} {:.4f} {:.4f} '
                      '{:.4f} {:.4f} {:.4f} {:.4f} {:.4f} {:.4f}'.format(
                          cols['name'][i], cols['alpha'][i], b[i][0], b[i][1], b[i][2],
                          b[i][3], dims[i][1], dims[i][2], dims[i][0], loc[i][0], loc[i][1],
                          loc[i][2], cols['rotation_y'][i], cols['score'][i]), file=fh)


def bbox2result_kitti(results, data_infos, class_names, submission_prefix=None,
                      pcd_limit_range=WAYMO_PCD_LIMIT_RANGE):
    """WaymoDataset.bbox2result_kitti, load_mode 'lidar_frame': per frame, the KITTI-format
    anno kitti_eval reads, built by slicing the device conversion's columns.  With
    ``submission_prefix``, writes ``<prefix>/<sample_idx:07d>.txt`` for every frame that
    keeps a box, as the reference does."""
    if len(results) > 0 and isinstance(results[0], dict) and 'pts_bbox' in results[0]:
        results = [r['pts_bbox'] for r in results]
    c = convert_set(results, data_infos, pcd_limit_range)
    cols, off = _kept_columns(c, class_names)
    if submission_prefix is not None:
        _write_submissions(submission_prefix, cols, off, data_infos)
    # np.stack of the reference's per-box lists: the name width is that of the frame's
    # longest name
    width = np.zeros(len(off) - 1, np.int64)
    nz = np.flatnonzero(np.diff(off) > 0)
    if len(nz):
        width[nz] = np.maximum.reduceat(cols['name_len'], off[:-1][nz])
    annos = []
    for f in range(len(off) - 1):
        s, e = int(off[f]), int(off[f + 1])
        if s == e:
            annos.append(_empty_anno())
            continue
        annos.append({'name': cols['name'][s:e].astype(f'<U{width[f]}'),
                      'truncated': np.zeros(e - s), 'occluded': np.zeros(e - s, np.int64),
                      'alpha': cols['alpha'][s:e], 'bbox': cols['bbox'][s:e],
                      'dimensions': cols['dimensions'][s:e], 'location': cols['location'][s:e],
                      'rotation_y': cols['rotation_y'][s:e], 'score': cols['score'][s:e],
                      'sample_idx': cols['sample_idx'][s:e]})
    return annos


def _metric_names(metric):
    names = [metric] if isinstance(metric, str) else list(metric)
    if any('waymo' in m for m in names):
        raise NotImplementedError(
            "metric 'waymo' (LET-3D-AP) runs Waymo's compute_detection_let_metrics_main "
            'binary: write the predictions with waymo_eval.write_objects and score them with '
            'the binary')
    if not any('kitti' in m for m in names):
        raise ValueError(f'invalid metric {metric!r}')


def gt_annos_of(data_infos, cam_sync=True):
    """WaymoDataset.load_annotations: ``cam_sync_annos`` replace ``annos`` when cam_sync is
    set and the infos hold annos."""
    if cam_sync and 'annos' in data_infos[0]:
        missing = [f for f, i in enumerate(data_infos) if 'cam_sync_annos' not in i]
        if missing:
            raise ValueError(f'cam_sync=True but data_infos[{missing[0]}] has no cam_sync_annos')
        return [i['cam_sync_annos'] for i in data_infos]
    missing = [f for f, i in enumerate(data_infos) if 'annos' not in i]
    if missing:
        raise ValueError(f'data_infos[{missing[0]}] has no annos')
    return [i['annos'] for i in data_infos]


def _score(results, data_infos, class_names, pcd_limit_range, gt, eval_types,
           submission_prefix, overlap_limit):
    """Converts and scores one result set."""
    from . import kitti_eval as ke
    dt, flags, rows = _detections(results, data_infos, class_names, pcd_limit_range, gt,
                                  submission_prefix)
    return ke.kitti_eval_columns(gt, dt, list(class_names), eval_types, f32_flags=flags,
                                 overlap_limit=overlap_limit, dt_rows=rows)


def _detections(results, data_infos, class_names, pcd_limit_range, gt, submission_prefix):
    """The kept detections as ``kitti_eval_columns`` takes them: host ``off`` / ``code`` /
    ``alpha``, the dtype flags, and the evaluator rows (fp64 bbox, alpha, location,
    dimensions, rotation_y, score), gathered on the device from the conversion's output."""
    import torch
    from . import kitti_eval as ke
    d = _convert(results, data_infos, pcd_limit_range)
    keep = d['keep'].bool()
    v = keep.cpu().numpy()
    labels = d['labels'][v].astype(np.int64)
    if len(labels) and (labels.min() < 0 or labels.max() >= len(class_names)):
        bad = labels[(labels < 0) | (labels >= len(class_names))][0]
        raise ValueError(f'label {int(bad)} has no class name')
    off = np.concatenate([[0], np.cumsum(v, dtype=np.int64)])[np.asarray(d['off'], np.int64)]
    if submission_prefix is not None:
        host = dict(d, keep=v, out=d['out'].cpu().numpy(),
                    sample_idx=d['sample_idx'].cpu().numpy())
        _write_submissions(submission_prefix, *_kept_columns(host, class_names), data_infos)
    scores = torch.from_numpy(d['scores']).to(keep.device)
    rows = torch.empty(len(labels), 13, dtype=torch.float64, device=keep.device)
    rows[:, :12] = d['out'][keep, :12]
    rows[:, 12] = scores[keep]
    dt = dict(off=off, code=ke.name_codes(np.asarray(list(class_names)), False)[labels],
              alpha=rows[:, 4].cpu().numpy().astype(np.float32))
    dtypes = {k: np.zeros(0, np.float32) for k in ke.DT_COLS}
    dtypes['score'] = np.zeros(0, d['scores'].dtype)
    flags = ke.column_f32_flags(gt, dtypes)
    if (np.diff(off) == 0).any():
        # an empty frame's anno holds float64 arrays, so the reference's concatenation of
        # the frames is float64
        flags &= ~(2 | 8 | 32)
    return dt, flags, rows


def evaluate(results, data_infos, class_names=WAYMO_CLASSES, metric='kitti',
             pcd_limit_range=WAYMO_PCD_LIMIT_RANGE, cam_sync=True, submission_prefix=None,
             return_str=False, overlap_limit=None):
    """WaymoDataset.evaluate with the KITTI metric, load_mode 'lidar_frame': the device
    conversion of every frame, then kitti_eval against ``cam_sync_annos`` (``annos`` with
    ``cam_sync=False``).  Plain per-frame results (what ``MultiViewDfM.simple_test`` returns)
    give kitti_eval's ret_dict as it is, with AOS where valid; results wrapped as
    ``{'pts_bbox': ...}`` are scored for BEV and 3-D with keys ``pts_bbox/<key>``, each value
    rounded as ``float('{:.4f}'.format(ap))``.  No ``KITTI/`` prefix is added.  With
    ``return_str`` the report string comes second.  ``overlap_limit`` bounds the evaluator's
    overlap buffer (bytes; see ``kitti_eval.KittiEvaluator``)."""
    from . import kitti_eval as ke
    _metric_names(metric)
    if len(results) != len(data_infos):
        raise ValueError(f'{len(results)} results but {len(data_infos)} data_infos')
    if len(results) == 0:
        raise ValueError('no results')
    gt = ke.concat_annos(gt_annos_of(data_infos, cam_sync), ('name',) + ke.GT_COLS)
    if isinstance(results[0], dict) and any(k in results[0] for k in
                                            ('pts_bbox', 'img_bbox', 'img_bbox2d')):
        ap_dict, strs = {}, []
        for name in results[0]:
            if '2d' in name:
                raise ValueError(f"'{name}' results (bbox2result_kitti2d) are not supported")
            prefix = None if submission_prefix is None else submission_prefix + name
            s, d = _score([r[name] for r in results], data_infos, class_names,
                          pcd_limit_range, gt, ['bev', '3d'], prefix, overlap_limit)
            ap_dict.update({f'{name}/{k}': float('{:.4f}'.format(v)) for k, v in d.items()})
            strs.append(f'Results of {name}:\n' + s)
        result_str = '\n'.join(strs)
    else:
        result_str, ap_dict = _score(results, data_infos, class_names, pcd_limit_range, gt,
                                     ['bbox', 'bev', '3d'], submission_prefix, overlap_limit)
    return (ap_dict, result_str) if return_str else ap_dict
