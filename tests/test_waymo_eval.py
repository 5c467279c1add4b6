"""Waymo camera-only LET-3D-AP building blocks: the Objects codec, the numpy restatement of
the pair stage against the binary's recorded decisions, and dfm_op_let_iou against it."""
import gzip
import json
import math
import os

import numpy as np
import pytest

from depth_from_motion_b200 import waymo_eval as W
from oracle import waymo_let_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


def _probes():
    with gzip.open(os.path.join(GOLDEN, 'waymo_let.json.gz'), 'rt') as f:
        return json.load(f)['probes']


def _objects():
    return np.load(os.path.join(GOLDEN, 'waymo_objects.npz'))


def _type_line(p):
    key = 'OBJECT_TYPE_TYPE_%s_LEVEL_2: ' % ('VEHICLE', 'PEDESTRIAN', 'SIGN', 'CYCLIST')[p['type'] - 1]
    return next(line for line in p['stdout'].splitlines() if line.startswith(key))


def _line_values(line):
    return [v for v in (line.split('LET-mAPL ')[1].split(']')[0],
                        line.split('LET-mAP ')[1].split(']')[0],
                        line.split('LET-mAPH ')[1].split(']')[0])]


# ---- codec -----------------------------------------------------------------------------
def test_read_objects_parses_protobuf_bytes():
    z = _objects()
    frames = W.read_objects(z['raw'].tobytes())
    assert len(frames) == int(z['frame'].max()) + 1
    box = np.concatenate([f['box'] for f in frames])
    np.testing.assert_array_equal(box, z['box'])
    np.testing.assert_array_equal(np.concatenate([f['camera_synced_box'] for f in frames]),
                                  z['synced'])
    np.testing.assert_array_equal(np.concatenate([f['type'] for f in frames]), z['type'])
    np.testing.assert_array_equal(np.concatenate([f['score'] for f in frames]), z['score'])
    np.testing.assert_array_equal(
        np.concatenate([f['detection_difficulty_level'] for f in frames]), z['difficulty'])
    np.testing.assert_array_equal(
        np.concatenate([f['num_lidar_points_in_box'] for f in frames]), z['num_points'])
    assert sum((f['most_visible_camera_name'] for f in frames), []) == list(z['camera'])
    assert sum((f['id'] for f in frames), []) == list(z['id'])


def test_write_objects_reproduces_protobuf_bytes(tmp_path):
    z = _objects()
    frames = W.read_objects(z['raw'].tobytes())
    assert W.objects_bytes(frames) == z['grouped'].tobytes()
    W.write_objects(tmp_path / 'o.bin', frames)
    assert (tmp_path / 'o.bin').read_bytes() == z['grouped'].tobytes()


def test_reference_gt_bin_parses():
    raw = _objects()['gt_bin'].tobytes()
    (fr,) = W.read_objects(raw)
    assert fr['context_name'] == '1071392229495085036_1844_790_1864_790'
    assert fr['frame_timestamp_micros'] == 1507315488219118
    assert fr['type'].tolist() == [1] and fr['num_lidar_points_in_box'].tolist() == [100]
    assert fr['score'].tolist() == [np.float32(0.8)]
    assert fr['box'][0, 0] == 69.676503339360735
    assert W.objects_bytes([fr]) == raw


def test_truncated_objects_raise():
    raw = _objects()['raw'].tobytes()
    with pytest.raises(ValueError):
        W.read_objects(raw[:-3])


# ---- the restatement against the binary ------------------------------------------------
def test_oracle_reproduces_binary_pair_decisions():
    for p in _probes():
        iou, aff, hacc = O.let_pair(p['pred'], p['gt'])
        apl, ap, aph = _line_values(_type_line(p))
        assert O.matchable(iou, aff, p['type']) == (ap == '1'), p
        g = np.subtract(p['gt'][:3], O.SENSOR)
        # a GT centre less than 1e-6 m from the sensor: the binary's affinity is not the
        # formula there (see the oracle), only the match decision is compared
        if ap == '1' and np.sqrt(g @ g) >= 1e-6:
            # the binary carries the weights in float32 and prints 6 significant digits
            assert abs(float(apl) - aff) <= 1e-6 and abs(float(aph) - hacc) <= 1e-6, p


def test_probes_record_every_breakdown_line():
    for p in _probes():
        lines = [ln for ln in p['stdout'].splitlines() if ': [LET-mAPL ' in ln]
        assert len(lines) == 36, p


def test_probes_cover_both_sides_of_every_threshold():
    kinds = {}
    for p in _probes():
        kinds.setdefault((p['kind'], p['type']), set()).add(_line_values(_type_line(p))[1])
    for t in (1, 2, 3, 4):
        assert kinds[('iou_threshold', t)] == {'0', '1'}
    assert kinds[('size_floor', 1)] == {'0', '1'}


# ---- device ----------------------------------------------------------------------------
def _degenerate_pairs():
    b = [20.0, 3.0, 0.5, 4.0, 2.0, 1.5, 0.3]
    shared = [20.0 + 4.0 * math.cos(0.3), 3.0 + 4.0 * math.sin(0.3), 0.5, 4.0, 2.0, 1.5, 0.3]
    return [
        (b, b),                                              # coincident
        (shared, b),                                         # shared edge
        ([20.0, 3.0, 2.0, 4.0, 2.0, 1.5, 0.3], b),           # zero z overlap (touching)
        ([20.0, 3.0, 5.0, 4.0, 2.0, 1.5, 0.3], b),           # disjoint in z
        ([1.43, 0.0, 2.18, 4.0, 2.0, 1.5, 0.0], [1.43, 0.0, 2.18, 4.0, 2.0, 1.5, 0.0]),
        ([2.0, 0.5, 2.0, 4.0, 2.0, 1.5, 1.0], [1.43, 0.0, 2.18, 4.0, 2.0, 1.5, 0.0]),
        ([20.0, 3.0, 0.5, 4.0, 2.0, 1.5, 0.3 + math.pi / 2], b),
        ([20.0, 3.0, 0.5, 4.0, 2.0, 1.5, 0.3 + 2 * math.pi], b),
        ([20.0, 3.0, 0.5, 0.0, 2.0, 1.5, 0.3], b),           # zero volume
        ([20.0, 3.0, 0.5, 4.0, 0.01, 1.5, 0.3], b),          # at the 0.01 m size floor
        # just above the floor, far from the origin: corners nearly collinear after rounding
        ([3.1e6, -2.7e6, 0.5, 0.0101, 0.0101, 1.5, 0.7], [3.1e6, -2.7e6, 0.5, 0.0102, 0.0101, 1.5, 0.7 + 1e-9]),
        ([3.1e6, -2.7e6, 0.5, 4.0, 0.0101, 1.5, 0.7], [3.1e6 + 1e-9, -2.7e6, 0.5, 4.0, 0.0102, 1.5, 0.7]),
    ]


@pytest.mark.gpu
def test_let_iou_matches_oracle_on_probes_and_degenerate_geometry():
    pairs = [(p['pred'], p['gt']) for p in _probes()] + _degenerate_pairs()
    pd = np.array([a for a, _ in pairs], np.float64)
    gt = np.array([b for _, b in pairs], np.float64)
    out = W.let_iou(pd, gt).cpu().numpy()
    assert out.shape == (len(pairs), len(pairs), 3)
    for i, (a, b) in enumerate(pairs):
        ref = O.let_pair(a, b)
        np.testing.assert_allclose(out[i, i], ref, rtol=0, atol=1e-12, err_msg=str((a, b)))
    # coincident boxes: IoU 1, affinity 1, heading accuracy 1
    n = len(_probes())
    np.testing.assert_allclose(out[n, n], (1.0, 1.0, 1.0), rtol=0, atol=1e-12)


@pytest.mark.gpu
def test_let_iou_all_pairs_and_matchable_agree_with_binary():
    rng = np.random.default_rng(7)
    probes = _probes()
    pd = np.array([p['pred'] for p in probes])
    gt = np.array([p['gt'] for p in probes])
    out = W.let_iou(pd, gt).cpu().numpy()
    for i in rng.choice(len(probes), 40, replace=False):
        for j in rng.choice(len(probes), 40, replace=False):
            np.testing.assert_allclose(out[i, j], O.let_pair(pd[i], gt[j]), rtol=0, atol=1e-12)
    m = W.matchable(out, [p['type'] for p in probes])
    for i, p in enumerate(probes):
        assert bool(m[i, i]) == (_line_values(_type_line(p))[1] == '1'), p


@pytest.mark.gpu
def test_let_iou_empty_and_invalid():
    import torch
    from depth_from_motion_b200 import capi
    assert tuple(W.let_iou(np.zeros((0, 7)), np.zeros((3, 7))).shape) == (0, 3, 3)
    with pytest.raises(RuntimeError):
        capi.check(capi.lib().dfm_op_let_iou(None, None, 1, 1, None, None), 'dfm_op_let_iou')
    x = torch.zeros(7, dtype=torch.float64, device='cuda')
    with pytest.raises(RuntimeError):
        capi.check(capi.lib().dfm_op_let_iou(x.data_ptr(), x.data_ptr(), 0, 1, x.data_ptr(),
                                             None), 'dfm_op_let_iou')
