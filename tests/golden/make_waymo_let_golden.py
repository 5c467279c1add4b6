"""Generates tests/golden/waymo_let.json.gz and waymo_objects.npz on the CPU from Waymo's
``compute_detection_let_metrics_main`` (the binary mmdet3d ships under
``mmdet3d/core/evaluation/waymo_utils``), run unchanged.

    python tests/golden/make_waymo_let_golden.py <reference checkout>

- Pair probes: one frame with one GT (camera_synced_box, FRONT, 10 points) and one
  prediction of the same type.  The binary's stdout is recorded verbatim (all 36
  breakdown lines).  In the OBJECT_TYPE line of the pair's type, with a single pair, LET-mAP is 1 when the pair matches and 0 otherwise, and a
  matched pair's mAPL / mAPH are its affinity / heading accuracy at 6 significant digits.
  The probes hold random pairs (those whose float32 LET-IoU lies within 1e-6 of the
  threshold are dropped), pairs bisected onto the IoU threshold of every type from both
  sides, the 0.5 m tolerance floor, GT at and within a micrometre of the sensor, and boxes
  at and around the 0.01 m size floor.
- Codec fixture: random ``Objects`` serialised by protobuf with message classes built from
  the descriptors embedded in the binary, and the reference's one-vehicle test ``gt.bin``.
"""
import gzip
import json
import math
import os
import random
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from depth_from_motion_b200 import waymo_eval as W  # noqa: E402
from oracle import waymo_let_oracle as O  # noqa: E402

TYPES = {1: 'VEHICLE', 2: 'PEDESTRIAN', 3: 'SIGN', 4: 'CYCLIST'}


def load_classes(binary):
    """Objects message class from the FileDescriptorProtos embedded in the binary."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    data = open(binary, 'rb').read()
    valid = {1: 2, 2: 2, 3: 2, 4: 2, 5: 2, 6: 2, 7: 2, 8: 2, 9: 2, 10: 0, 11: 0, 12: 2, 14: 0}

    def walk(i):
        s = i
        while i < len(data):
            tag, j = W._read_varint(data, i)
            f, wt = tag >> 3, tag & 7
            if valid.get(f) != wt:
                break
            if wt == 0:
                _, j = W._read_varint(data, j)
            else:
                ln, j = W._read_varint(data, j)
                j += ln
            i = j
        return data[s:i]
    fds = {}
    for m in re.finditer(rb'\n.(waymo_open_dataset/[a-z_/]+\.proto)\x12', data):
        fd = descriptor_pb2.FileDescriptorProto.FromString(walk(m.start()))
        fds[fd.name] = fd
    pool = descriptor_pool.DescriptorPool()
    done = set()

    def add(name):
        if name in done:
            return
        for d in fds[name].dependency:
            add(d)
        pool.Add(fds[name])
        done.add(name)
    for n in fds:
        add(n)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName('waymo.open_dataset.Objects'))


def gt_frame(box, t):
    return {'context_name': 'probe', 'frame_timestamp_micros': 1,
            'box': np.zeros((1, 7)), 'camera_synced_box': np.array([box], np.float64),
            'type': np.array([t], np.int32), 'score': np.ones(1, np.float32), 'id': [''],
            'detection_difficulty_level': np.array([2], np.int32),
            'num_lidar_points_in_box': np.array([10], np.int32),
            'most_visible_camera_name': ['FRONT'],
            'has': np.array([W.HAS_LABEL | W.HAS_BOX | W.HAS_TYPE | W.HAS_DIFFICULTY |
                             W.HAS_NUM_POINTS | W.HAS_CAMERA | W.HAS_SYNCED_BOX], np.int32)}


def pd_frame(box, t):
    return {'context_name': 'probe', 'frame_timestamp_micros': 1,
            'box': np.array([box], np.float64), 'type': np.array([t], np.int32),
            'score': np.array([0.9], np.float32)}


def run(binary, gt, pd):
    with tempfile.TemporaryDirectory() as d:
        g, p = os.path.join(d, 'gt.bin'), os.path.join(d, 'pd.bin')
        W.write_objects(g, gt)
        W.write_objects(p, pd)
        return subprocess.run([binary, p, g], capture_output=True, text=True,
                              check=True).stdout


def type_line(stdout, t):
    key = f'OBJECT_TYPE_TYPE_{TYPES[t]}_LEVEL_2: '
    return next(line for line in stdout.splitlines() if line.startswith(key))


def probe_stdout(binary, gbox, pbox, t):
    return run(binary, [gt_frame(gbox, t)], [pd_frame(pbox, t)])


def matched(line):
    return float(re.search(r'LET-mAP (\S+)\]', line).group(1)) > 0.5


def main(ref):
    binary = os.path.join(ref, 'mmdet3d/core/evaluation/waymo_utils/'
                               'compute_detection_let_metrics_main')
    rnd = random.Random(20261016)
    probes = []
    # random pairs around a GT
    while len(probes) < 160:
        t = rnd.choice([1, 1, 2, 3, 4])
        r, az = rnd.uniform(2, 70), rnd.uniform(-math.pi, math.pi)
        size = {1: (4.5, 2.0, 1.6), 2: (0.9, 0.9, 1.8), 3: (0.6, 0.2, 0.8), 4: (1.8, 0.8, 1.7)}[t]
        g = [r * math.cos(az), r * math.sin(az), rnd.uniform(-1, 1.5), *size,
             rnd.uniform(-math.pi, math.pi)]
        s = rnd.uniform(0.7, 1.3)
        p = [g[0] + rnd.gauss(0, 0.08 * r ** 0.5), g[1] + rnd.gauss(0, 0.08 * r ** 0.5),
             g[2] + rnd.gauss(0, 0.15), g[3] * s, g[4] * rnd.uniform(0.8, 1.2),
             g[5] * rnd.uniform(0.8, 1.2), g[6] + rnd.gauss(0, 0.4)]
        iou, aff, _ = O.let_pair(p, g)
        if abs(float(np.float32(iou)) - float(O.IOU_THR[t])) < 1e-6:
            continue
        probes.append({'gt': g, 'pred': p, 'type': t, 'kind': 'random'})
    # bisected onto each type's IoU threshold (lateral shift) and the affinity edge
    for t in (1, 2, 3, 4):
        g = [20.0, 0.0, 0.0, 4.0, 2.0, 1.5, 0.0]
        lo, hi = 0.0, 2.0
        for _ in range(40):
            mid = (lo + hi) / 2
            if matched(type_line(probe_stdout(binary, g, [20.5, mid, 0.0, 4.0, 2.0, 1.5, 0.0],
                                              t), t)):
                lo = mid
            else:
                hi = mid
        for y in (lo, hi):
            probes.append({'gt': g, 'pred': [20.5, y, 0.0, 4.0, 2.0, 1.5, 0.0], 'type': t,
                           'kind': 'iou_threshold'})
    for x in (3.0, 3.2, 3.49, 3.6):  # GT at 3 m: 0.5 m tolerance floor
        probes.append({'gt': [3.0, 0, 0, 4, 2, 1.5, 0], 'pred': [x, 0, 0, 4, 2, 1.5, 0.1],
                       'type': 1, 'kind': 'tolerance_floor'})
    probes.append({'gt': [1.43, 0, 2.18, 4, 2, 1.5, 0], 'pred': [1.43, 0, 2.18, 4, 2, 1.5, 0],
                   'type': 1, 'kind': 'gt_at_sensor'})
    probes.append({'gt': [20, 0, 0, 4, 2, 1.5, 0], 'pred': [21, 0, 0, 4, 2, 1.5, 0.1],
                   'type': 1, 'kind': 'shift_and_heading'})
    # GT centre within a micrometre of the sensor: the binary's affinity departs from the
    # formula by up to 2e-5 there (at 1e-6 m and beyond it follows the formula)
    for dx in (0.0, 1e-9, 1e-6, 1e-3):
        for off in (0.0, 0.01):
            g = [1.43 + dx, 0.0, 2.18, 4, 2, 1.5, 0]
            probes.append({'gt': g, 'pred': [g[0] + off] + g[1:], 'type': 1,
                           'kind': 'near_sensor'})
    # boxes a few nanometres thin, far from the origin (corners collinear to rounding), and
    # identical boxes at and just above the 0.01 m size floor of every dimension
    for dims in ((4.0, 0.01, 1.5), (0.01, 2.0, 1.5), (4.0, 2.0, 0.01), (4.0, 0.0105, 1.5),
                 (0.0105, 2.0, 1.5), (4.0, 2.0, 0.0105)):
        g = [20.0, 0.0, 0.4, *dims, 0.0]
        probes.append({'gt': g, 'pred': list(g), 'type': 1, 'kind': 'size_floor'})
    for t, (ln, wd) in ((1, (4.0, 3e-9)), (1, (3e-9, 2.0)), (2, (3e-9, 3e-9))):
        g = [61.7, -23.3, 0.4, ln, wd, 1.5, 0.7]
        for p in (g, [61.7 + 1e-9, -23.3, 0.4, ln, wd * 1.5, 1.5, 0.7 + 1e-7],
                  [61.8, -23.2, 0.4, 4.0, 2.0, 1.5, 0.7]):
            probes.append({'gt': g, 'pred': list(p), 'type': t, 'kind': 'thin_box'})
    for pr in probes:
        pr['stdout'] = probe_stdout(binary, pr['gt'], pr['pred'], pr['type'])
    with gzip.GzipFile(os.path.join(HERE, 'waymo_let.json.gz'), 'wb', mtime=0) as f:
        f.write(json.dumps({'generator': 'tests/golden/make_waymo_let_golden.py',
                            'binary': 'compute_detection_let_metrics_main', 'probes': probes},
                           indent=1).encode())

    # codec fixture
    Objects = load_classes(binary)
    m = Objects()
    for k in range(60):
        o = m.objects.add()
        o.context_name = f'segment-{k % 4}'
        o.frame_timestamp_micros = 1507315488219118 + 100000 * (k % 3)
        if rnd.random() < 0.8:
            o.score = rnd.random()
        lab = o.object
        vals = [rnd.uniform(-80, 80), rnd.uniform(-80, 80), rnd.uniform(-2, 3),
                rnd.uniform(0.5, 5), rnd.uniform(0.5, 2.5), rnd.uniform(0.5, 3),
                rnd.uniform(-math.pi, math.pi)]
        b = lab.box
        b.center_x, b.center_y, b.center_z, b.length, b.width, b.height, b.heading = vals
        lab.type = rnd.randint(0, 4)
        if rnd.random() < 0.5:
            lab.id = f'obj{k}'
        if rnd.random() < 0.5:
            lab.detection_difficulty_level = rnd.randint(0, 2)
        if rnd.random() < 0.6:
            lab.num_lidar_points_in_box = rnd.randint(0, 40)
        if rnd.random() < 0.6:
            lab.most_visible_camera_name = rnd.choice(['FRONT', 'FRONT_LEFT', 'SIDE_RIGHT', ''])
        if rnd.random() < 0.6:
            lab.camera_synced_box.CopyFrom(b)
            lab.camera_synced_box.center_x += 0.25
        if rnd.random() < 0.3:
            lab.tracking_difficulty_level = 1     # a field the codec skips
    raw = m.SerializeToString()
    # the same objects in frame order, without the skipped field: what write_objects emits
    keys = []
    for o in m.objects:
        if (o.context_name, o.frame_timestamp_micros) not in keys:
            keys.append((o.context_name, o.frame_timestamp_micros))
    grouped = Objects()
    for key in keys:
        for o in m.objects:
            if (o.context_name, o.frame_timestamp_micros) == key:
                c = grouped.objects.add()
                c.CopyFrom(o)
                c.object.ClearField('tracking_difficulty_level')
    gtbin = open(os.path.join(ref, 'tests/data/waymo/waymo_format/gt.bin'), 'rb').read()
    arrays = {'raw': np.frombuffer(raw, np.uint8), 'grouped': np.frombuffer(
        grouped.SerializeToString(), np.uint8), 'gt_bin': np.frombuffer(gtbin, np.uint8)}
    fields = {
        'box': [[o.object.box.center_x, o.object.box.center_y, o.object.box.center_z,
                 o.object.box.length, o.object.box.width, o.object.box.height,
                 o.object.box.heading] for o in grouped.objects],
        'synced': [[o.object.camera_synced_box.center_x, o.object.camera_synced_box.center_y,
                    o.object.camera_synced_box.center_z, o.object.camera_synced_box.length,
                    o.object.camera_synced_box.width, o.object.camera_synced_box.height,
                    o.object.camera_synced_box.heading] for o in grouped.objects],
        'type': [o.object.type for o in grouped.objects],
        'score': [o.score for o in grouped.objects],
        'difficulty': [o.object.detection_difficulty_level for o in grouped.objects],
        'num_points': [o.object.num_lidar_points_in_box for o in grouped.objects]}
    for k, v in fields.items():
        arrays[k] = np.asarray(v, np.float32 if k == 'score' else None)
    arrays['camera'] = np.array([o.object.most_visible_camera_name for o in grouped.objects])
    arrays['id'] = np.array([o.object.id for o in grouped.objects])
    arrays['frame'] = np.array([keys.index((o.context_name, o.frame_timestamp_micros))
                                for o in grouped.objects])
    np.savez_compressed(os.path.join(HERE, 'waymo_objects.npz'), **arrays)


if __name__ == '__main__':
    main(sys.argv[1])
