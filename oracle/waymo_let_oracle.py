"""Plain numpy restatement of the pair stage of Waymo's camera-only LET-3D-AP, as
``compute_detection_let_metrics_main`` computes it (the binary mmdet3d's
``WaymoDataset.evaluate`` runs for the camsync configs).

Each rule was pinned against that binary with probe files:

- The prediction is aligned along the ray from the sensor to its centre, to the point of
  that ray closest to the GT centre (``align``).  LET-IoU is the 3-D IoU of the aligned
  prediction and the GT: the BEV rectangles clipped against each other, times the z
  overlap, over the union volume.  It is 0 when either box has a length, width or height
  of 0.01 m or less.  The binary rounds it to float32 before comparing it
  with the type's threshold (0.5 vehicle, 0.3 pedestrian, sign and cyclist).
- The longitudinal error is the offset's projection on the unit vector from the sensor to
  the GT centre; the tolerance is ``max(0.1 * |c_gt - s|, 0.5)`` and the affinity
  ``1 - min(|e_lon| / tol, 1)``.  APL weighs a TP by it.  The binary follows this formula
  for GT centres 1e-6 m or more from the sensor.  Closer in it does not: a GT at the sensor
  scores 0.999998 against an identical prediction, and a GT 1e-9 m from it scores 0.999982
  against a prediction 0.01 m further out, where the formula gives 0.98.  The binary
  seems to regularise the unit vector there; this restatement does not model it, and no
  real GT lies within a micrometre of the roof-mounted sensor.
- The heading accuracy is ``1 - |wrapped heading error| / pi``.  APH weighs a TP by it
  alone, not by its product with the affinity.
"""
import math

import numpy as np

SENSOR = (1.43, 0.0, 2.18)
LON_TOL_PCT = 0.1
LON_TOL_MIN = 0.5
# a box with a dimension at or below this has LET-IoU 0 with every box
MIN_BOX_DIM = 0.01
# IoU threshold per type (UNKNOWN, VEHICLE, PEDESTRIAN, SIGN, CYCLIST), float32 as the
# binary's config stores them
IOU_THR = np.array([0.0, 0.5, 0.3, 0.3, 0.3], np.float32)


# ---- geometry ------------------------------------------------------------------------
def bev_corners(b):
    """Counter-clockwise BEV corners of box b = (x, y, z, length, width, height, heading)."""
    c, s = math.cos(b[6]), math.sin(b[6])
    hl, hw = b[3] / 2.0, b[4] / 2.0
    out = []
    for dx, dy in ((hl, hw), (-hl, hw), (-hl, -hw), (hl, -hw)):
        out.append((b[0] + dx * c - dy * s, b[1] + dx * s + dy * c))
    return out


def _clip(poly, a, b):
    """Sutherland-Hodgman: the part of convex polygon poly left of the directed edge a->b."""
    out = []
    n = len(poly)
    for i in range(n):
        p, q = poly[i], poly[(i + 1) % n]
        sp = (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0])
        sq = (b[0] - a[0]) * (q[1] - a[1]) - (b[1] - a[1]) * (q[0] - a[0])
        if sp >= 0:
            out.append(p)
        if (sp >= 0) != (sq >= 0):
            t = sp / (sp - sq)
            out.append((p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])))
    return out


def _area(poly):
    s = 0.0
    for i in range(len(poly)):
        p, q = poly[i], poly[(i + 1) % len(poly)]
        s += p[0] * q[1] - q[0] * p[1]
    return 0.5 * s


def iou3d(a, b):
    """fp64 3-D IoU of two boxes rotated about z (0 when either has a dimension of
    MIN_BOX_DIM or less)."""
    if min(a[3], a[4], a[5], b[3], b[4], b[5]) <= MIN_BOX_DIM:
        return 0.0
    va = a[3] * a[4] * a[5]
    vb = b[3] * b[4] * b[5]
    zo = min(a[2] + a[5] / 2, b[2] + b[5] / 2) - max(a[2] - a[5] / 2, b[2] - b[5] / 2)
    if zo <= 0:
        return 0.0
    poly = bev_corners(a)
    cb = bev_corners(b)
    for i in range(4):
        if len(poly) < 3:
            return 0.0
        poly = _clip(poly, cb[i], cb[(i + 1) % 4])
    if len(poly) < 3:
        return 0.0
    inter = max(_area(poly), 0.0) * zo
    u = va + vb - inter
    return inter / u if u > 0 else 0.0


def _dot3(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _sub3(a, b):
    return (float(a[0]) - float(b[0]), float(a[1]) - float(b[1]), float(a[2]) - float(b[2]))


def align(pd, gt):
    """The prediction moved along the sensor -> prediction ray to the point of that ray
    closest to the GT centre."""
    out = [float(x) for x in pd]
    v = _sub3(pd, SENSOR)
    n2 = _dot3(v, v)
    if n2 > 0.0:
        t = _dot3(_sub3(gt, SENSOR), v) / n2
        out[:3] = [float(SENSOR[c]) + t * v[c] for c in range(3)]
    return out


def affinity(pd, gt):
    g = _sub3(gt, SENSOR)
    rg = math.sqrt(_dot3(g, g))
    tol = max(LON_TOL_PCT * rg, LON_TOL_MIN)
    e = _dot3(_sub3(pd, gt), g) / rg if rg > 0.0 else 0.0
    return 1.0 - min(abs(e) / tol, 1.0)


def heading_accuracy(pd, gt):
    d = abs(float(pd[6]) - float(gt[6]))
    d = math.fmod(d, 2 * math.pi)
    d = min(d, 2 * math.pi - d)
    return 1.0 - d / math.pi


def let_pair(pd, gt):
    """(LET-IoU, affinity, heading accuracy) of prediction box pd and GT box gt."""
    return iou3d(align(pd, gt), gt), affinity(pd, gt), heading_accuracy(pd, gt)


def matchable(iou, aff, gt_type):
    """Whether a same-type pair can match: affinity > 0 and float32(LET-IoU) >= the
    threshold of the GT's type."""
    return aff > 0.0 and np.float32(iou) >= IOU_THR[int(gt_type)]
