"""Building blocks of Waymo's camera-only LET-3D-AP (``WaymoDataset.evaluate(metric='waymo')``
with ``cam_sync=True``, which runs Waymo's ``compute_detection_let_metrics_main``).

- ``read_objects`` / ``write_objects``: a pure-Python protobuf wire codec for the fields of
  ``metrics_pb2.Objects`` the metric reads, so a ``cam_gt.bin`` can be read and a
  submission ``.bin`` written without TensorFlow or the Waymo package.  The writer emits the
  bytes protobuf's serialiser emits for the same set fields.
- ``let_iou``: the metric's pair stage on the device (``csrc/waymo_eval_kernels.cuh``): the
  longitudinal alignment, the fp64 3-D rotated IoU, the longitudinal affinity and the
  heading accuracy of every (prediction, GT) pair.
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
