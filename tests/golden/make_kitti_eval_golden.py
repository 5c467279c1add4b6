"""Writes tests/golden/kitti_eval.npz + kitti_eval.json: the KITTI evaluator of mmdet3d
(core/evaluation/kitti_utils/eval.py and rotate_iou.py, executed verbatim through
oracle/ref_loader) on 200 frames built from demo/data/kitti/kitti_000008_infos.pkl.

numba.cuda runs in its simulator (NUMBA_ENABLE_CUDASIM=1), which evaluates math.cos / sin
and the scalar temporaries of the rotated IoU in float64. Its overlaps are therefore a few
ulp away from numba on a GPU, not bitwise equal. So that every matching decision is
unambiguous, detections whose overlap with any GT (or, for the 2-D metric, any DontCare
box) lies within 1e-4 of a min-overlap are dropped before the evaluation is recorded.

Stored: the inputs (CSR per frame), the overlaps of each metric in [dt, gt] order per frame,
and for each configuration (metric, class, difficulty, overlap set) the TP scores as
get_thresholds receives them, the thresholds, the pr counts and precision / recall / aos;
plus ret_dict and result_str.

Run from the repository root: python tests/golden/make_kitti_eval_golden.py
"""
import json
import os
import pickle
import sys
import types

os.environ['NUMBA_ENABLE_CUDASIM'] = '1'
import numpy as np  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from oracle import ref_loader  # noqa: E402

KU = 'mmdet3d/core/evaluation/kitti_utils/'
NAMES = ('Car', 'Pedestrian', 'Cyclist', 'Van', 'Person_sitting')
MIN_OVERLAPS = (0.7, 0.5, 0.25)
MARGIN = 1e-4


def load_eval():
    pkg = types.ModuleType('ku_ref')
    pkg.__path__ = [os.path.join(ref_loader.REFERENCE_ROOT, KU)]
    sys.modules['ku_ref'] = pkg
    ref_loader._exec('ku_ref.rotate_iou', KU + 'rotate_iou.py')
    return ref_loader._exec('ku_ref.eval', KU + 'eval.py')


def make_frames(num_frames, seed=0):
    with open(os.path.join(ref_loader.REFERENCE_ROOT,
                           'demo/data/kitti/kitti_000008_infos.pkl'), 'rb') as f:
        base = pickle.load(f)[0]['annos']
    rng = np.random.default_rng(seed)
    keys = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location',
            'rotation_y')
    gts, dts = [], []
    for _ in range(num_frames):
        g = {k: base[k].copy() for k in keys}
        n = len(g['name'])
        real = g['name'] != 'DontCare'
        # relabel objects over the five named classes, vary occlusion / truncation / size
        names = g['name'].astype('<U14')
        names[real] = rng.choice(NAMES, real.sum(), p=(0.5, 0.2, 0.15, 0.1, 0.05))
        g['name'] = names
        g['occluded'] = np.where(real, rng.integers(0, 3, n), g['occluded'])
        g['truncated'] = np.where(real, rng.choice((0.0, 0.1, 0.2, 0.4, 0.6), n),
                                  g['truncated'])
        shift = rng.normal(0, 1.5, (n, 3)) * real[:, None]
        g['location'] = g['location'] + shift
        g['bbox'] = g['bbox'] + rng.normal(0, 8, (n, 4)) * real[:, None]
        g['bbox'][:, 3] = np.maximum(g['bbox'][:, 3], g['bbox'][:, 1] + 1)
        g['rotation_y'] = g['rotation_y'] + rng.normal(0, 0.3, n) * real
        g['alpha'] = g['alpha'] + rng.normal(0, 0.3, n) * real
        keep = rng.uniform(size=n) > 0.1
        if rng.uniform() < 0.05:   # a few frames without GT at all
            keep[:] = False
        g = {k: v[keep] for k, v in g.items()}
        # detections: jittered objects (some relabelled) and false positives
        src = np.flatnonzero(g['name'] != 'DontCare')
        src = src[rng.uniform(size=len(src)) > 0.15]
        nfp = int(rng.integers(0, 4))
        m = len(src) + nfp
        d = {}
        d['name'] = np.concatenate([
            np.where(rng.uniform(size=len(src)) < 0.9, g['name'][src],
                     rng.choice(NAMES[:3], len(src))),
            rng.choice(NAMES[:3], nfp)]).astype('<U14')
        fp_loc = np.stack([rng.uniform(-15, 15, nfp), rng.uniform(1, 2, nfp),
                           rng.uniform(5, 50, nfp)], 1)
        fp_dim = np.stack([rng.uniform(0.5, 4.5, nfp), rng.uniform(1.4, 2.0, nfp),
                           rng.uniform(0.5, 2.0, nfp)], 1)
        x0 = rng.uniform(0, 1100, nfp)
        y0 = rng.uniform(100, 300, nfp)
        fp_box = np.stack([x0, y0, x0 + rng.uniform(10, 200, nfp),
                           y0 + rng.uniform(10, 120, nfp)], 1)
        sig = rng.uniform(0.05, 0.6, len(src))[:, None]
        d['location'] = np.concatenate([g['location'][src] + rng.normal(0, 1, (len(src), 3))
                                        * sig, fp_loc])
        d['dimensions'] = np.concatenate([g['dimensions'][src] * (1 + rng.normal(
            0, 0.1, (len(src), 3))), fp_dim])
        d['rotation_y'] = np.concatenate([g['rotation_y'][src] + rng.normal(0, 0.2, len(src)),
                                          rng.uniform(-np.pi, np.pi, nfp)])
        d['bbox'] = np.concatenate([g['bbox'][src] + rng.normal(0, 10, (len(src), 4)) * sig,
                                    fp_box])
        d['alpha'] = np.concatenate([g['alpha'][src] + rng.normal(0, 0.3, len(src)),
                                     rng.uniform(-np.pi, np.pi, nfp)])
        d['score'] = rng.uniform(0, 1, m).round(2)   # coarse scores: ties occur
        if rng.uniform() < 0.05:   # a few frames without detections
            d = {k: v[:0] for k, v in d.items()}
        gts.append(g)
        dts.append(d)
    return gts, dts


def near_boundary(ev, gts, dts):
    """[(frame, dt index)] whose overlap lies within MARGIN of a min-overlap."""
    bad = set()
    for metric in range(3):
        ovs = ev.calculate_iou_partly(dts, gts, metric)[0]
        for f, ov in enumerate(ovs):
            for j in np.flatnonzero(np.any(np.abs(ov[..., None] - MIN_OVERLAPS) < MARGIN,
                                           axis=(1, 2))):
                bad.add((f, int(j)))
    for f, (g, d) in enumerate(zip(gts, dts)):
        dc = g['bbox'][g['name'] == 'DontCare']
        if len(dc) and len(d['bbox']):
            ov = ev.image_box_overlap(d['bbox'], dc, 0)
            for j in np.flatnonzero(np.any(np.abs(ov[..., None] - MIN_OVERLAPS) < MARGIN,
                                           axis=(1, 2))):
                bad.add((f, int(j)))
    return bad


def pack(annos, with_score):
    off = np.cumsum([0] + [len(a['name']) for a in annos]).astype(np.int64)
    cat = lambda k, w: np.concatenate([a[k].reshape(-1, w) for a in annos]).astype(np.float64)
    out = dict(off=off, name=np.concatenate([a['name'] for a in annos]).astype('<U14'),
               alpha=cat('alpha', 1)[:, 0], bbox=cat('bbox', 4), dimensions=cat('dimensions', 3),
               location=cat('location', 3), rotation_y=cat('rotation_y', 1)[:, 0])
    if with_score:
        out['score'] = cat('score', 1)[:, 0]
    else:
        out['occluded'] = cat('occluded', 1)[:, 0]
        out['truncated'] = cat('truncated', 1)[:, 0]
    return out


def main(num_frames=200):
    ev = load_eval()
    gts, dts = make_frames(num_frames)
    while True:
        bad = near_boundary(ev, gts, dts)
        if not bad:
            break
        for f in {f for f, _ in bad}:
            keep = np.ones(len(dts[f]['name']), bool)
            keep[[j for g, j in bad if g == f]] = False
            dts[f] = {k: v[keep] for k, v in dts[f].items()}
    arrays = {}
    for prefix, annos, ws in (('gt', gts, False), ('dt', dts, True)):
        for k, v in pack(annos, ws).items():
            arrays[f'{prefix}_{k}'] = v
    for metric in range(3):
        ovs = ev.calculate_iou_partly(dts, gts, metric)[0]
        arrays[f'overlap{metric}'] = np.concatenate([o.reshape(-1) for o in ovs]).astype(
            np.float64)

    # record every intermediate of eval_class through its module-level callees
    rec = {'thr_in': [], 'thr_out': [], 'pr': [], 'eval': []}
    get_thresholds, fused, eval_class = ev.get_thresholds, ev.fused_compute_statistics, \
        ev.eval_class

    def rec_thresholds(scores, num_gt, num_sample_pts=41):
        rec['thr_in'].append((np.sort(scores)[::-1].copy(), int(num_gt)))
        out = get_thresholds(scores, num_gt, num_sample_pts)
        rec['thr_out'].append(np.array(out, np.float64))
        return out

    def rec_fused(overlaps, pr, *a, **k):
        if not rec['pr'] or rec['pr'][-1] is not pr:
            rec['pr'].append(pr)
        return fused(overlaps, pr, *a, **k)

    def rec_eval_class(*a, **k):
        r = eval_class(*a, **k)
        rec['eval'].append({n: v.copy() for n, v in r.items()})
        return r

    ev.get_thresholds, ev.fused_compute_statistics, ev.eval_class = \
        rec_thresholds, rec_fused, rec_eval_class
    classes = ['Car', 'Pedestrian', 'Cyclist']
    result_str, ret_dict = ev.kitti_eval(gts, dts, list(classes))
    assert len(rec['eval']) == 3 and len(rec['thr_in']) == 3 * 3 * 3 * 2
    # configurations in evaluation order: metric, class, difficulty, overlap set
    nc = len(rec['thr_in'])
    arrays['thr_num_gt'] = np.array([n for _, n in rec['thr_in']], np.int64)
    arrays['tp_off'] = np.cumsum([0] + [len(s) for s, _ in rec['thr_in']]).astype(np.int64)
    arrays['tp_scores'] = np.concatenate([s for s, _ in rec['thr_in']]).astype(np.float64)
    arrays['thr_count'] = np.array([len(t) for t in rec['thr_out']], np.int64)
    thr = np.zeros((nc, 41))
    pr = np.zeros((nc, 41, 4))
    for c in range(nc):
        thr[c, :len(rec['thr_out'][c])] = rec['thr_out'][c]
    # pr arrays of configurations with no thresholds are never passed to fused_compute_
    # statistics' loop body but are still created; match them up by the threshold count
    it = iter(rec['pr'])
    for c in range(nc):
        p = next(it)
        assert len(p) == arrays['thr_count'][c]
        pr[c, :len(p)] = p
    arrays['thresholds'] = thr
    arrays['pr'] = pr
    for n in ('precision', 'recall', 'orientation'):
        arrays[n] = np.stack([e[n] for e in rec['eval']])   # [metric][cls][diff][k][41]
    np.savez_compressed(os.path.join(HERE, 'kitti_eval.npz'), **arrays)
    with open(os.path.join(HERE, 'kitti_eval.json'), 'w') as f:
        json.dump({'classes': classes, 'result_str': result_str,
                   'ret_dict': {k: float(v) for k, v in ret_dict.items()}}, f, indent=1)
    print(result_str)


if __name__ == '__main__':
    main()
