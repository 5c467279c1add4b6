"""Host restatement of the KITTI evaluator (mmdet3d kitti_utils/eval.py + rotate_iou.py), our
own code, one frame and one box pair at a time.

The rotated IoU is written op for op with numpy float32 scalars where numba types the
reference's arithmetic as float32, and Python floats (float64) where a float64 literal or an
integer enters, so it is the bitwise target of the device kernel.  The one input it cannot
restate is libdevice's cosf / sinf; by default it takes float32(cos(float64(angle))), and a
caller may pass the device's own values (``trig``).

``evaluate`` returns every intermediate the device evaluator exposes: overlaps per metric,
TP scores, thresholds and pr counts per configuration, in the configuration
order ((metric slot * classes + class slot) * 3 + difficulty) * 2 + overlap set.
"""
import math

import numpy as np

F = np.float32
MIN_HEIGHT = (40, 25, 25)
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
CLASS_NAMES = ('car', 'pedestrian', 'cyclist')


# ---------------------------------------------------------------- rotated IoU (float32)
def _corners(r, trig):
    c, s = trig
    hx, hy = F(r[2] / F(2)), F(r[3] / F(2))
    cx = (-hx, -hx, hx, hx)
    cy = (-hy, hy, hy, -hy)
    out = []
    for i in range(4):
        out.append(F(F(c * cx[i]) + F(s * cy[i])) + r[0])
        out.append(F(F(-s * cx[i]) + F(c * cy[i])) + r[1])
    return [F(v) for v in out]


def _in_quad(px, py, c):
    ab0, ab1 = c[2] - c[0], c[3] - c[1]
    ad0, ad1 = c[6] - c[0], c[7] - c[1]
    ap0, ap1 = px - c[0], py - c[1]
    abab = ab0 * ab0 + ab1 * ab1
    abap = ab0 * ap0 + ab1 * ap1
    adad = ad0 * ad0 + ad1 * ad1
    adap = ad0 * ap0 + ad1 * ap1
    return abab >= abap and abap >= 0 and adad >= adap and adap >= 0


def _seg(p1, p2, i, j):
    A0, A1 = p1[2 * i], p1[2 * i + 1]
    B0, B1 = p1[2 * ((i + 1) % 4)], p1[2 * ((i + 1) % 4) + 1]
    C0, C1 = p2[2 * j], p2[2 * j + 1]
    D0, D1 = p2[2 * ((j + 1) % 4)], p2[2 * ((j + 1) % 4) + 1]
    BA0, BA1 = B0 - A0, B1 - A1
    DA0, CA0 = D0 - A0, C0 - A0
    DA1, CA1 = D1 - A1, C1 - A1
    acd = DA1 * CA0 > CA1 * DA0
    bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0)
    if acd != bcd:
        abc = CA1 * BA0 > BA1 * CA0
        abd = DA1 * BA0 > BA1 * DA0
        if abc != abd:
            DC0, DC1 = D0 - C0, D1 - C1
            ABBA = A0 * B1 - B0 * A1
            CDDC = C0 * D1 - D0 * C1
            DH = BA1 * DC0 - BA0 * DC1
            Dx = ABBA * DC0 - BA0 * CDDC
            Dy = ABBA * DC1 - BA1 * CDDC
            with np.errstate(divide='ignore', invalid='ignore'):
                return F(Dx / DH), F(Dy / DH)
    return None


def default_trig(angle):
    a = float(F(angle))
    return F(math.cos(a)), F(math.sin(a))


def rotated_inter(r1, r2, trig1=None, trig2=None):
    r1 = [F(v) for v in r1]
    r2 = [F(v) for v in r2]
    c1 = _corners(r1, trig1 or default_trig(r1[4]))
    c2 = _corners(r2, trig2 or default_trig(r2[4]))
    pts = []
    for i in range(4):
        if _in_quad(c1[2 * i], c1[2 * i + 1], c2):
            pts.append([c1[2 * i], c1[2 * i + 1]])
        if _in_quad(c2[2 * i], c2[2 * i + 1], c1):
            pts.append([c2[2 * i], c2[2 * i + 1]])
    for i in range(4):
        for j in range(4):
            t = _seg(c1, c2, i, j)
            if t is not None:
                pts.append(list(t))
    n = len(pts)
    if n > 0:
        sx, sy = F(0), F(0)
        for p in pts:
            sx = F(sx + p[0])
            sy = F(sy + p[1])
        cx, cy = F(float(sx) / n), F(float(sy) / n)
        vs = []
        with np.errstate(divide='ignore', invalid='ignore'):
            for p in pts:
                v0, v1 = F(p[0] - cx), F(p[1] - cy)
                d = F(np.sqrt(F(F(v0 * v0) + F(v1 * v1))))
                v0, v1 = F(v0 / d), F(v1 / d)
                if v1 < 0:
                    v0 = F(-2.0 - float(v0))
                vs.append(v0)
        for i in range(1, n):
            if vs[i - 1] > vs[i]:
                temp, tp = vs[i], pts[i]
                j = i
                while j > 0 and vs[j - 1] > temp:
                    vs[j] = vs[j - 1]
                    pts[j] = pts[j - 1]
                    j -= 1
                vs[j] = temp
                pts[j] = tp
    area = 0.0
    for i in range(n - 2):
        a, b, c = pts[0], pts[i + 1], pts[i + 2]
        cr = F(F((a[0] - c[0]) * (b[1] - c[1])) - F((a[1] - c[1]) * (b[0] - c[0])))
        area = area + abs(float(cr) / 2.0)
    return area


def rotate_iou_eval_pair(r1, r2, criterion=-1, trig1=None, trig2=None):
    """devRotateIoUEval(r1, r2, criterion) as stored in its float32 output."""
    area1 = F(F(r1[2]) * F(r1[3]))
    area2 = F(F(r2[2]) * F(r2[3]))
    inter = rotated_inter(r1, r2, trig1, trig2)
    with np.errstate(divide='ignore', invalid='ignore'):
        if criterion == -1:
            den = float(F(area1 + area2)) - inter
            v = inter / den if den != 0 else (math.nan if inter == 0 else math.copysign(
                math.inf, inter) * math.copysign(1.0, den))
        elif criterion in (0, 1):
            a = float(area1 if criterion == 0 else area2)
            v = inter / a if a != 0 else (math.nan if inter == 0 else math.inf)
        else:
            v = inter
    return F(v)


def rotate_iou_eval(boxes, qboxes, criterion=-1, trig=None, qtrig=None):
    """rotate_iou_gpu_eval: iou[n][k] = devRotateIoUEval(qboxes[k], boxes[n], criterion).
    trig / qtrig: optional (cos, sin) float32 arrays per box."""
    boxes = np.asarray(boxes, np.float64).astype(np.float32)
    qboxes = np.asarray(qboxes, np.float64).astype(np.float32)
    out = np.zeros((len(boxes), len(qboxes)), np.float32)
    for n in range(len(boxes)):
        for k in range(len(qboxes)):
            out[n, k] = rotate_iou_eval_pair(
                qboxes[k], boxes[n], criterion,
                None if qtrig is None else (F(qtrig[0][k]), F(qtrig[1][k])),
                None if trig is None else (F(trig[0][n]), F(trig[1][n])))
    return out


# ---------------------------------------------------------------- 2-D and 3-D overlaps
def image_box_overlap(boxes, query_boxes, criterion=-1):
    """image_box_overlap with numpy's dtype rules for float32 / float64 inputs."""
    TB, TQ = boxes.dtype.type, query_boxes.dtype.type
    TP = np.result_type(boxes.dtype, query_boxes.dtype).type
    out = np.zeros((len(boxes), len(query_boxes)), boxes.dtype)
    for k in range(len(query_boxes)):
        q = query_boxes[k]
        qarea = TQ((q[2] - q[0]) * (q[3] - q[1]))
        for n in range(len(boxes)):
            b = boxes[n]
            iw = TP(min(TP(b[2]), TP(q[2])) - max(TP(b[0]), TP(q[0])))
            if iw > 0:
                ih = TP(min(TP(b[3]), TP(q[3])) - max(TP(b[1]), TP(q[1])))
                if ih > 0:
                    barea = TB((b[2] - b[0]) * (b[3] - b[1]))
                    if criterion == -1:
                        ua = TP(TP(TP(barea) + TP(qarea)) - TP(iw * ih))
                    elif criterion == 0:
                        ua = TP(barea)
                    elif criterion == 1:
                        ua = TP(qarea)
                    else:
                        ua = TP(1)
                    out[n, k] = TP(TP(iw * ih) / ua)
    return out


def d3_box_overlap(boxes, qboxes, trig=None, qtrig=None):
    """d3_box_overlap(boxes, qboxes) with criterion -1: float32 output."""
    rinc = rotate_iou_eval(boxes[:, [0, 2, 3, 5, 6]], qboxes[:, [0, 2, 3, 5, 6]], 2, trig, qtrig)
    TB, TQ = boxes.dtype.type, qboxes.dtype.type
    TP = np.result_type(boxes.dtype, qboxes.dtype).type
    for i in range(len(boxes)):
        for j in range(len(qboxes)):
            if rinc[i, j] > 0:
                b, q = boxes[i], qboxes[j]
                iw = TP(min(TP(b[1]), TP(q[1])) - max(TP(TB(b[1] - b[4])), TP(TQ(q[1] - q[4]))))
                if iw > 0:
                    area1 = TB(TB(b[3] * b[4]) * b[5])
                    area2 = TQ(TQ(q[3] * q[4]) * q[5])
                    inc = TP(iw * TP(rinc[i, j]))
                    ua = TP(TP(TP(area1) + TP(area2)) - inc)
                    rinc[i, j] = np.float32(inc / ua)
                else:
                    rinc[i, j] = 0.0
    return rinc


def frame_overlaps(g, d, metric, trig=None):
    """[dt, gt] overlaps of one frame, as float64 values of the reference's array.  trig:
    optional ((cos, sin) of the detections' yaws, (cos, sin) of the GT yaws) as float32."""
    dtrig, gtrig = trig if trig is not None else (None, None)
    if metric == 0:
        return image_box_overlap(np.asarray(d['bbox']), np.asarray(g['bbox'])).astype(np.float64)
    box = lambda a, cols: np.concatenate([np.asarray(a['location'])[:, cols],
                                          np.asarray(a['dimensions'])[:, cols],
                                          np.asarray(a['rotation_y'])[:, None]], 1)
    if metric == 1:
        return rotate_iou_eval(box(d, [0, 2]), box(g, [0, 2]), -1, dtrig, gtrig).astype(
            np.float64)
    return d3_box_overlap(box(d, [0, 1, 2]), box(g, [0, 1, 2]), dtrig, gtrig).astype(
        np.float64)


# ---------------------------------------------------------------- matching and counts
def clean_data(g, d, current_class, difficulty):
    name = CLASS_NAMES[current_class]
    ignored_gt, ignored_dt, dc = [], [], []
    num_valid = 0
    for i in range(len(g['name'])):
        bbox = g['bbox'][i]
        gname = str(g['name'][i]).lower()
        height = bbox[3] - bbox[1]
        if gname == name:
            vc = 1
        elif (name == 'pedestrian' and gname == 'person_sitting') or \
                (name == 'car' and gname == 'van'):
            vc = 0
        else:
            vc = -1
        ignore = (g['occluded'][i] > MAX_OCCLUSION[difficulty] or
                  g['truncated'][i] > MAX_TRUNCATION[difficulty] or
                  height <= MIN_HEIGHT[difficulty])
        if vc == 1 and not ignore:
            ignored_gt.append(0)
            num_valid += 1
        elif vc == 0 or (ignore and vc == 1):
            ignored_gt.append(1)
        else:
            ignored_gt.append(-1)
        if g['name'][i] == 'DontCare':
            dc.append(g['bbox'][i])
    for j in range(len(d['name'])):
        height = abs(d['bbox'][j][3] - d['bbox'][j][1])
        if height < MIN_HEIGHT[difficulty]:
            ignored_dt.append(1)
        elif str(d['name'][j]).lower() == name:
            ignored_dt.append(0)
        else:
            ignored_dt.append(-1)
    dc = np.stack(dc, 0).astype(np.float64) if dc else np.zeros((0, 4))
    return num_valid, ignored_gt, ignored_dt, dc


def compute_statistics(ov, g, d, ig, idt, dc, metric, min_overlap, thresh=0.0,
                       compute_fp=False, compute_aos=False, dt_data=None):
    nd, ng = len(idt), len(ig)
    scores = np.asarray(d['score'])
    assigned = [False] * nd
    below = [compute_fp and scores[j] < thresh for j in range(nd)]
    NO = -10000000.0
    tp = fp = fn = 0
    tps, deltas = [], []
    for i in range(ng):
        if ig[i] == -1:
            continue
        det, valid, max_ov, ass_ign = -1, NO, 0.0, False
        for j in range(nd):
            if idt[j] == -1 or assigned[j] or below[j]:
                continue
            o = ov[j, i]
            if not compute_fp and o > min_overlap and scores[j] > valid:
                det, valid = j, scores[j]
            elif compute_fp and o > min_overlap and (o > max_ov or ass_ign) and idt[j] == 0:
                max_ov, det, valid, ass_ign = o, j, 1, False
            elif compute_fp and o > min_overlap and valid == NO and idt[j] == 1:
                det, valid, ass_ign = j, 1, True
        if valid == NO and ig[i] == 0:
            fn += 1
        elif valid != NO and (ig[i] == 1 or idt[det] == 1):
            assigned[det] = True
        elif valid != NO:
            tp += 1
            tps.append(float(scores[det]))
            if compute_aos:
                deltas.append(float(dt_data[1][i] - dt_data[0][det]))
            assigned[det] = True
    sim = 0.0
    if compute_fp:
        for j in range(nd):
            if not (assigned[j] or idt[j] == -1 or idt[j] == 1 or below[j]):
                fp += 1
        nstuff = 0
        if metric == 0 and len(dc):
            ov_dc = image_box_overlap(dt_data[2], dc, 0)
            for i in range(len(dc)):
                for j in range(nd):
                    if assigned[j] or idt[j] in (-1, 1) or below[j]:
                        continue
                    if ov_dc[j, i] > min_overlap:
                        assigned[j] = True
                        nstuff += 1
        fp -= nstuff
        if compute_aos and (tp > 0 or fp > 0):
            for x in deltas:
                sim = sim + (1.0 + np.cos(x)) / 2.0
    return tp, fp, fn, sim, tps


def get_thresholds(scores, num_gt, num_sample_pts=41):
    scores = np.sort(np.asarray(scores, np.float64))[::-1]
    current_recall, out = 0.0, []
    for i, score in enumerate(scores):
        l_recall = (i + 1) / num_gt
        r_recall = (i + 2) / num_gt if i < len(scores) - 1 else l_recall
        if (r_recall - current_recall) < (current_recall - l_recall) and i < len(scores) - 1:
            continue
        out.append(score)
        current_recall += 1 / (num_sample_pts - 1.0)
    return np.array(out, np.float64), scores


def evaluate(gt_annos, dt_annos, classes, metrics, compute_aos, min_overlaps, overlaps=None):
    """pr [configs][41][4], threshold counts, thresholds [configs][41], sorted TP scores per
    config and overlaps per metric (lists of per-frame [dt, gt] arrays).  ``min_overlaps`` is
    kitti_eval's [2][3][5] table; ``overlaps`` may be given per metric."""
    N = len(gt_annos)
    ovs = {}
    for m in metrics:
        ovs[m] = overlaps[m] if overlaps is not None else [
            frame_overlaps(gt_annos[f], dt_annos[f], m) for f in range(N)]
    nc = len(metrics) * len(classes) * 6
    pr = np.zeros((nc, 41, 4))
    thr = np.zeros((nc, 41))
    cnt = np.zeros(nc, np.int64)
    sorted_scores = []
    dt_data = []
    for f in range(N):
        dd = np.concatenate([np.asarray(dt_annos[f]['bbox']),
                             np.asarray(dt_annos[f]['alpha'])[:, None],
                             np.asarray(dt_annos[f]['score'])[:, None]], 1)
        gd = np.concatenate([np.asarray(gt_annos[f]['bbox']),
                             np.asarray(gt_annos[f]['alpha'])[:, None]], 1)
        dt_data.append((dd[:, 4], gd[:, 4], dd[:, :4]))
    for ms, m in enumerate(metrics):
        for cs, c in enumerate(classes):
            for diff in range(3):
                prep = [clean_data(gt_annos[f], dt_annos[f], c, diff) for f in range(N)]
                num_valid = sum(p[0] for p in prep)
                for k in range(2):
                    cfg = ((ms * len(classes) + cs) * 3 + diff) * 2 + k
                    mo = min_overlaps[k, m, c]
                    tps = []
                    for f in range(N):
                        _, ig, idt, dc = prep[f]
                        tps += compute_statistics(ovs[m][f], gt_annos[f], dt_annos[f], ig, idt,
                                                  dc, m, mo)[4]
                    t, ss = get_thresholds(tps, num_valid)
                    sorted_scores.append(ss)
                    cnt[cfg] = len(t)
                    thr[cfg, :len(t)] = t
                    for f in range(N):
                        _, ig, idt, dc = prep[f]
                        for ti, th in enumerate(t):
                            tp, fp, fn, sim, _ = compute_statistics(
                                ovs[m][f], gt_annos[f], dt_annos[f], ig, idt, dc, m, mo, th,
                                True, compute_aos and m == 0, dt_data[f])
                            pr[cfg, ti, 0] += tp
                            pr[cfg, ti, 1] += fp
                            pr[cfg, ti, 2] += fn
                            pr[cfg, ti, 3] += sim
    return dict(pr=pr, thr_count=cnt, thresholds=thr, tp_scores=sorted_scores, overlaps=ovs)
