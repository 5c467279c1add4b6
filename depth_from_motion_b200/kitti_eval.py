"""KITTI evaluation on the H100: ``kitti_eval`` of mmdet3d (core/evaluation/kitti_utils/eval.py)
with its matching, thresholds and counts in ``csrc/kitti_eval_kernels.cuh``.

The GPU computes, for every (metric, class, difficulty, overlap set), the pr counts of each
threshold in one sequence of launches; precision, recall, AOS and AP11 / AP40 are then taken
on the host from those [configs x 41] arrays exactly as eval_class / do_eval / kitti_eval do,
including the report string and the ``KITTI/...`` keys.
"""
import ctypes

import numpy as np

from . import capi

CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting'}
NAME_TO_CLASS = {v: n for n, v in CLASS_TO_NAME.items()}
# gt / dt class ids of the device inputs: clean_data compares lower-cased names
CODE_OF_NAME = {'car': 0, 'pedestrian': 1, 'cyclist': 2, 'van': 3, 'person_sitting': 4}
CODE_OTHER, CODE_DONTCARE = 7, 8
METRICS = ('bbox', 'bev', '3d')
N_SAMPLE_PTS = 41
# [overlap set][metric][class], kitti_eval's tables
OVERLAP_0_7 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5], [0.7, 0.5, 0.5, 0.7, 0.5],
                        [0.7, 0.5, 0.5, 0.7, 0.5]])
OVERLAP_0_5 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25],
                        [0.5, 0.25, 0.25, 0.5, 0.25]])
MIN_OVERLAPS = np.stack([OVERLAP_0_7, OVERLAP_0_5], axis=0)
GT_KEYS = ('name', 'alpha', 'bbox', 'location', 'dimensions', 'rotation_y', 'occluded',
           'truncated')
DT_KEYS = ('name', 'alpha', 'bbox', 'location', 'dimensions', 'rotation_y', 'score')
MAX_DT_PER_FRAME = 1024


def class_ids(current_classes):
    """kitti_eval's class argument (a name, an int, or a list of them) -> list of ints."""
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    out = []
    for c in current_classes:
        if isinstance(c, str):
            if c not in NAME_TO_CLASS:
                raise ValueError(f'unknown class {c!r}')
            c = NAME_TO_CLASS[c]
        c = int(c)
        if c not in (0, 1, 2):
            # clean_data indexes ['car', 'pedestrian', 'cyclist'] with the class id
            raise ValueError(f'class {CLASS_TO_NAME.get(c, c)} cannot be evaluated: the KITTI '
                             'difficulty rules exist for Car, Pedestrian and Cyclist only')
        out.append(c)
    if not out:
        raise ValueError('no class to evaluate')
    if len(out) > 3:
        raise ValueError(f'{len(out)} classes given; at most 3 (Car, Pedestrian, Cyclist)')
    return out


def _check_annos(annos, keys, what):
    for f, a in enumerate(annos):
        missing = [k for k in keys if k not in a]
        if missing:
            raise ValueError(f'{what}[{f}] lacks {missing}')
        n = len(a['name'])
        for k in keys:
            v = np.asarray(a[k])
            w = {'bbox': 4, 'location': 3, 'dimensions': 3}.get(k)
            if (v.shape != (n, w)) if w else (v.shape != (n,)):
                raise ValueError(f'{what}[{f}][{k!r}] has shape {v.shape} for {n} boxes')


def _is_f32(annos, keys):
    """True when numpy would hold the concatenation of these arrays as float32."""
    dts = [np.asarray(a[k]).dtype for a in annos for k in keys]
    return bool(dts) and np.result_type(*dts) == np.float32


def compute_aos_flag(gt_annos, dt_annos):
    """kitti_eval's rule: AOS only when some predicted alpha and the GT alphas are valid."""
    pred_alpha = any(np.asarray(a['alpha'])[np.asarray(a['alpha']) != -10].shape[0] != 0
                     for a in dt_annos)
    valid_alpha_gt = False
    for a in gt_annos:
        if len(a['alpha']) == 0:
            raise ValueError('a GT frame without boxes comes before the first frame with '
                             'boxes: the reference reads its alpha[0] and fails')
        if a['alpha'][0] != -10:
            valid_alpha_gt = True
            break
    return pred_alpha and valid_alpha_gt


def compute_aos_flag_columns(gt, dt):
    """``compute_aos_flag`` of sets in column form (see ``pack_columns``)."""
    pred_alpha = bool(np.any(np.asarray(dt['alpha']) != -10))
    off = np.asarray(gt['off'], np.int64)
    ng = np.diff(off)
    alpha = np.asarray(gt['alpha'])
    first = np.full(len(ng), -10.0)
    first[ng > 0] = alpha[off[:-1][ng > 0]]
    stop = (ng == 0) | (first != -10)   # the reference's loop ends at the first of these
    if not stop.any():
        return False
    if ng[int(np.argmax(stop))] == 0:
        raise ValueError('a GT frame without boxes comes before the first frame with boxes: '
                         'the reference reads its alpha[0] and fails')
    return pred_alpha


def name_codes(names, gt):
    """Device class codes of an array of names: clean_data's lower-cased comparisons, one
    vectorised comparison per class name."""
    names = np.asarray(names)
    codes = np.full(len(names), CODE_OTHER, np.int32)
    if len(names) == 0:
        return codes
    names = names.astype(str)
    done = np.zeros(len(names), bool)
    for n, c in CODE_OF_NAME.items():   # the spellings KITTI and Waymo annos use
        m = names == CLASS_TO_NAME[c]
        codes[m] = c
        done |= m
    rest = np.flatnonzero(~done)        # any other spelling: lower-cased, once per name
    if len(rest):
        uniq, inv = np.unique(names[rest], return_inverse=True)
        codes[rest] = np.array([CODE_OF_NAME.get(n.lower(), CODE_OTHER) for n in uniq],
                               np.int32)[inv.reshape(-1)]
    if gt:
        codes[names == 'DontCare'] |= CODE_DONTCARE
    return codes


GT_COLS = ('bbox', 'alpha', 'location', 'dimensions', 'rotation_y', 'occluded', 'truncated')
DT_COLS = ('bbox', 'alpha', 'location', 'dimensions', 'rotation_y', 'score')
_WIDTH = {'bbox': 4, 'location': 3, 'dimensions': 3}


def _columns(c, cols, what, values=True):
    off = np.asarray(c['off'], np.int64)
    if off.ndim != 1 or len(off) < 2 or off[0] != 0 or np.any(np.diff(off) < 0):
        raise ValueError(f'{what}: off must be ascending from 0 with one entry per frame + 1')
    n = int(off[-1])
    if n >= 1 << 31:
        raise ValueError(f'{what}: {n} boxes, more than the int32 offsets index')
    if not values:   # the caller has the rows: check the class column only
        cols = ()
    # one fp64 row per box, each column written into place once
    flat = np.empty((n, sum(_WIDTH.get(k, 1) for k in cols)), np.float64)
    j = 0
    for k in (('code',) if 'code' in c else ('name',)) + cols:
        if k not in c:
            raise ValueError(f'{what} lacks {k!r}')
        v = np.asarray(c[k])
        w = _WIDTH.get(k)
        if (v.shape != (n, w)) if w else (v.shape != (n,)):
            raise ValueError(f'{what}[{k!r}] has shape {v.shape} for {n} boxes')
        if k not in ('name', 'code'):
            flat[:, j:j + (w or 1)] = v.reshape(n, w or 1)
            j += w or 1
    return off, flat


def column_f32_flags(gt, dt):
    """``pack``'s dtype flags of sets in column form: a group is float32 when all its
    columns are."""
    f32 = lambda c, keys: all(np.asarray(c[k]).dtype == np.float32 for k in keys)
    return (f32(gt, ('bbox',)) * 1 | f32(dt, ('bbox',)) * 2 |
            f32(gt, ('location', 'dimensions', 'rotation_y')) * 4 |
            f32(dt, ('location', 'dimensions', 'rotation_y')) * 8 |
            f32(gt, ('bbox', 'alpha')) * 16 | f32(dt, ('bbox', 'alpha', 'score')) * 32)


def pack_columns(gt, dt, f32_flags=None, dt_rows=None):
    """Flat fp64 inputs of the device evaluator from sets in column form: ``gt`` / ``dt`` are
    dicts of the anno keys concatenated over frames (``name``, ``bbox`` [n, 4], ...) plus
    ``off`` [frames + 1], each frame's first box.  An int32 ``code`` column (``name_codes``
    of the names) may stand in for ``name``.  ``f32_flags`` (see ``pack``) defaults to the
    columns' own dtypes: a column group is float32 when all its columns are.  ``dt_rows``, an
    fp64 [detections, 13] array or CUDA tensor in the device layout (bbox, alpha, location,
    dimensions, rotation_y, score), stands in for dt's value columns (``dt`` then needs only
    ``off``, ``name`` or ``code``, and the flags)."""
    g_off, g = _columns(gt, GT_COLS, 'gt')
    d_off, d = _columns(dt, DT_COLS, 'dt', values=dt_rows is None)
    if dt_rows is not None:
        if f32_flags is None:
            raise ValueError('dt_rows needs f32_flags')
        if tuple(dt_rows.shape) != (int(d_off[-1]), 13):
            raise ValueError(f'dt_rows has shape {tuple(dt_rows.shape)} for {int(d_off[-1])} '
                             'detections')
        d = dt_rows
    if len(g_off) != len(d_off):
        raise ValueError(f'{len(g_off) - 1} GT frames but {len(d_off) - 1} detection frames')
    nd = np.diff(d_off)
    if nd.size and nd.max() > MAX_DT_PER_FRAME:
        f = int(np.argmax(nd))
        raise ValueError(f'dt frame {f} holds {int(nd[f])} detections, more than '
                         f'{MAX_DT_PER_FRAME}')
    if f32_flags is None:
        f32_flags = column_f32_flags(gt, dt)
    ng = np.diff(g_off)
    code = lambda c, is_gt: (np.asarray(c['code'], np.int32) if 'code' in c else
                             name_codes(c['name'], is_gt))
    return dict(gt=g, dt=d, gt_code=code(gt, True), dt_code=code(dt, False),
                gt_off=g_off.astype(np.int32),
                dt_off=d_off.astype(np.int32),
                pair_off=np.concatenate([[0], np.cumsum(ng * nd)]).astype(np.int64),
                f32_flags=int(f32_flags))


def concat_annos(annos, keys):
    """Per-frame anno dicts -> one dict of concatenated columns plus ``off``."""
    out = {'off': np.concatenate([[0], np.cumsum([len(a['name']) for a in annos])])}
    for k in keys:
        w = _WIDTH.get(k)
        out[k] = np.concatenate([np.asarray(a[k]).reshape(-1, w) if w else
                                 np.asarray(a[k]).reshape(-1) for a in annos])
    return out


def pack(gt_annos, dt_annos):
    """Flat fp64 inputs of the device evaluator plus the dtype flags."""
    if len(gt_annos) != len(dt_annos):
        raise ValueError(f'{len(gt_annos)} GT frames but {len(dt_annos)} detection frames')
    if len(gt_annos) == 0:
        raise ValueError('no frames to evaluate')
    _check_annos(gt_annos, GT_KEYS, 'gt_annos')
    _check_annos(dt_annos, DT_KEYS, 'dt_annos')
    for f, a in enumerate(dt_annos):
        if len(a['name']) > MAX_DT_PER_FRAME:
            raise ValueError(f'dt_annos[{f}] holds {len(a["name"])} detections, more than '
                             f'{MAX_DT_PER_FRAME}')
    flags = (_is_f32(gt_annos, ('bbox',)) * 1 | _is_f32(dt_annos, ('bbox',)) * 2 |
             _is_f32(gt_annos, ('location', 'dimensions', 'rotation_y')) * 4 |
             _is_f32(dt_annos, ('location', 'dimensions', 'rotation_y')) * 8 |
             _is_f32(gt_annos, ('bbox', 'alpha')) * 16 |
             _is_f32(dt_annos, ('bbox', 'alpha', 'score')) * 32)
    return pack_columns(concat_annos(gt_annos, ('name',) + GT_COLS),
                        concat_annos(dt_annos, ('name',) + DT_COLS), flags)


class KittiEvaluator:
    """Owns one ``dfm_kitti_eval`` handle for a (classes, metrics, aos) setting."""

    def __init__(self, classes, metrics, compute_aos, overlap_limit=None):
        self.classes, self.metrics = list(classes), list(metrics)
        self.compute_aos = bool(compute_aos)
        self.overlap_limit = overlap_limit   # bytes of one part's overlaps; None: the default
        self.f32_flags = None
        self._h = None

    def _handle(self, f32_flags):
        if self._h is not None and f32_flags == self.f32_flags:
            return self._h
        self.close()
        d = capi.KittiEvalDesc()
        d.num_classes = len(self.classes)
        d.num_metrics = len(self.metrics)
        for i, c in enumerate(self.classes):
            d.classes[i] = c
        for i, m in enumerate(self.metrics):
            d.metrics[i] = m
        d.compute_aos = int(self.compute_aos)
        d.f32_flags = f32_flags
        for ms, m in enumerate(self.metrics):
            for cs, c in enumerate(self.classes):
                for k in range(2):
                    d.min_overlap[(ms * 3 + cs) * 2 + k] = MIN_OVERLAPS[k, m, c]
        h = ctypes.c_void_p()
        capi.check(capi.lib().dfm_kitti_eval_create(ctypes.byref(d), ctypes.byref(h)),
                   'dfm_kitti_eval_create')
        self._h, self.f32_flags = h, f32_flags
        if self.overlap_limit is not None:
            capi.check(capi.lib().dfm_kitti_eval_set_overlap_limit(h, int(self.overlap_limit)),
                       'dfm_kitti_eval_set_overlap_limit')
        return h

    def workspace(self):
        """The last forward's (workspace bytes, overlap buffer bytes, number of parts)."""
        w, o, n = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
        capi.check(capi.lib().dfm_kitti_eval_workspace(self._h, ctypes.byref(w), ctypes.byref(o),
                                                       ctypes.byref(n)),
                   'dfm_kitti_eval_workspace')
        return w.value, o.value, n.value

    @property
    def num_configs(self):
        return len(self.metrics) * len(self.classes) * 6

    def forward(self, packed, keep=False):
        """pr [configs][41][4] and threshold counts [configs] (numpy) of the packed inputs."""
        import torch
        h = self._handle(packed['f32_flags'])
        dev = torch.device('cuda')
        t = {k: (v if isinstance(v, torch.Tensor) else torch.from_numpy(v)).to(dev)
             for k, v in packed.items() if isinstance(v, (np.ndarray, torch.Tensor))}
        nc = self.num_configs
        pr = torch.empty(nc, N_SAMPLE_PTS, 4, dtype=torch.float64, device=dev)
        cnt = torch.empty(nc, dtype=torch.int32, device=dev)
        status = torch.empty(1, dtype=torch.int32, device=dev)
        p = lambda x: ctypes.c_void_p(x.data_ptr()) if x.numel() else None
        stream = torch.cuda.current_stream().cuda_stream
        capi.check(capi.lib().dfm_kitti_eval_forward(
            h, len(packed['gt_off']) - 1, len(packed['gt']), len(packed['dt']),
            int(packed['pair_off'][-1]), p(t['gt']), p(t['gt_code']), p(t['gt_off']),
            p(t['dt']), p(t['dt_code']), p(t['dt_off']), p(t['pair_off']), p(pr), p(cnt),
            p(status), ctypes.c_void_p(stream)), 'dfm_kitti_eval_forward')
        if keep:
            self._inputs = t   # the debug hook reads device state that refers to them
        pr_h, cnt_h = pr.cpu().numpy(), cnt.cpu().numpy()
        if int(status.item()) != 0:
            raise RuntimeError(f'dfm_kitti_eval_forward: a frame holds more than '
                               f'{MAX_DT_PER_FRAME} detections')
        if (cnt_h > N_SAMPLE_PTS).any():
            raise ValueError('a configuration yields more than 41 thresholds; the reference '
                             'fails on it')
        return pr_h, cnt_h

    def debug_tensor(self, name, numel, dtype):
        import torch
        out = torch.empty(numel, dtype=dtype, device='cuda')
        capi.check(capi.lib().dfm_kitti_eval_debug_tensor(
            self._h, name.encode(), ctypes.c_void_p(out.data_ptr()), numel,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
            'dfm_kitti_eval_debug_tensor')
        return out.cpu().numpy()

    def close(self):
        if self._h is not None:
            capi.lib().dfm_kitti_eval_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def precision_recall(pr, thr_count, num_classes, metric_aos):
    """eval_class's final loops: [classes][3][2][41] recall / precision / aos of one metric
    from its pr [classes * 3 * 2][41][4] and threshold counts."""
    shape = (num_classes, 3, 2, N_SAMPLE_PTS)
    precision, recall, aos = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    for c in range(num_classes * 6):
        m, idx_l, k = c // 6, (c // 2) % 3, c % 2
        n = int(thr_count[c])
        p = pr[c]
        with np.errstate(divide='ignore', invalid='ignore'):
            for i in range(n):
                recall[m, idx_l, k, i] = p[i, 0] / (p[i, 0] + p[i, 2])
                precision[m, idx_l, k, i] = p[i, 0] / (p[i, 0] + p[i, 1])
                if metric_aos:
                    aos[m, idx_l, k, i] = p[i, 3] / (p[i, 0] + p[i, 1])
        for i in range(n):
            precision[m, idx_l, k, i] = np.max(precision[m, idx_l, k, i:], axis=-1)
            recall[m, idx_l, k, i] = np.max(recall[m, idx_l, k, i:], axis=-1)
            if metric_aos:
                aos[m, idx_l, k, i] = np.max(aos[m, idx_l, k, i:], axis=-1)
    return {'recall': recall, 'precision': precision, 'orientation': aos}


def get_mAP11(prec):
    sums = 0
    for i in range(0, prec.shape[-1], 4):
        sums = sums + prec[..., i]
    return sums / 11 * 100


def get_mAP40(prec):
    sums = 0
    for i in range(1, prec.shape[-1]):
        sums = sums + prec[..., i]
    return sums / 40 * 100


def report(classes, eval_types, compute_aos, rets):
    """kitti_eval's result string and ret_dict from eval_class's output per metric
    (``rets[metric]``, metric 0 / 1 / 2)."""
    min_overlaps = MIN_OVERLAPS[:, :, classes]
    ap = {}
    for m, name in enumerate(METRICS):
        if name in eval_types:
            ap[name] = (get_mAP11(rets[m]['precision']), get_mAP40(rets[m]['precision']))
    if compute_aos:
        ap['aos'] = (get_mAP11(rets[0]['orientation']), get_mAP40(rets[0]['orientation']))
    rows = (('bbox', 'bbox', '2D'), ('bev', 'bev ', 'BEV'), ('3d', '3d  ', '3D'))
    difficulty = ['easy', 'moderate', 'hard']
    result, ret_dict = '', {}
    for a, tag in ((0, 'AP11'), (1, 'AP40')):
        result += f'\n----------- {tag} Results ------------\n\n'
        for j, curcls in enumerate(classes):
            curcls_name = CLASS_TO_NAME[curcls]
            for i in range(min_overlaps.shape[0]):
                result += ('{} {}@{:.2f}, {:.2f}, {:.2f}:\n'.format(curcls_name, tag,
                                                                    *min_overlaps[i, :, j]))
                for key, label, _ in rows:
                    if key in ap:
                        result += (label + ' ' + tag + ':{:.4f}, {:.4f}, {:.4f}\n').format(
                            *ap[key][a][j, :, i])
                if compute_aos:
                    result += ('aos  ' + tag + ':{:.2f}, {:.2f}, {:.2f}\n').format(
                        *ap['aos'][a][j, :, i])
                for idx in range(3):
                    postfix = f'{difficulty[idx]}_strict' if i == 0 else \
                        f'{difficulty[idx]}_loose'
                    prefix = f'KITTI/{curcls_name}'
                    for key, _, kname in rows[::-1]:
                        if key in ap:
                            ret_dict[f'{prefix}_{kname}_{tag}_{postfix}'] = ap[key][a][j, idx, i]
        if len(classes) > 1:
            result += '\nOverall {}@{}, {}, {}:\n'.format(tag, *difficulty)
            mean = {k: v[a].mean(axis=0) for k, v in ap.items()}
            for key, label, _ in rows:
                if key in mean:
                    result += (label + ' ' + tag + ':{:.4f}, {:.4f}, {:.4f}\n').format(
                        *mean[key][:, 0])
            if compute_aos:
                result += ('aos  ' + tag + ':{:.2f}, {:.2f}, {:.2f}\n').format(
                    *mean['aos'][:, 0])
            for idx in range(3):
                for key, _, kname in rows[::-1]:
                    if key in mean:
                        ret_dict[f'KITTI/Overall_{kname}_{tag}_{difficulty[idx]}'] = \
                            mean[key][idx, 0]
    return result, ret_dict


def check_eval_types(eval_types):
    eval_types = list(eval_types)
    if len(eval_types) == 0:
        raise ValueError('must contain at least one evaluation type')
    unknown = [t for t in eval_types if t not in METRICS + ('aos',)]
    if unknown:
        raise ValueError(f'unknown evaluation types {unknown}')
    if 'aos' in eval_types and 'bbox' not in eval_types:
        raise ValueError('must evaluate bbox when evaluating aos')
    return eval_types


def kitti_eval(gt_annos, dt_annos, current_classes, eval_types=('bbox', 'bev', '3d'),
               return_intermediates=False):
    """mmdet3d's ``kitti_eval``: returns ``(result_str, ret_dict)``.

    gt_annos / dt_annos: per frame, dicts of numpy arrays as ``kitti_infos_*.pkl`` /
    ``bbox2result_kitti`` hold them.  Classes are names or ints (Car, Pedestrian, Cyclist).
    With ``return_intermediates`` a third element holds the pr counts, threshold counts and
    eval_class outputs per metric.
    """
    eval_types = check_eval_types(eval_types)
    classes = class_ids(current_classes)
    packed = pack(gt_annos, dt_annos)
    compute_aos = compute_aos_flag(gt_annos, dt_annos)
    return _evaluate_packed(packed, classes, eval_types, compute_aos, return_intermediates)


def kitti_eval_columns(gt, dt, current_classes, eval_types=('bbox', 'bev', '3d'),
                       return_intermediates=False, f32_flags=None, overlap_limit=None,
                       dt_rows=None):
    """``kitti_eval`` of sets in column form (see ``pack_columns``): the same results as
    ``kitti_eval`` of the per-frame annos, without a Python loop over frames or boxes.
    ``overlap_limit`` bounds the bytes of one part's overlaps (see ``KittiEvaluator``);
    ``dt_rows`` see ``pack_columns``."""
    eval_types = check_eval_types(eval_types)
    classes = class_ids(current_classes)
    packed = pack_columns(gt, dt, f32_flags, dt_rows)
    compute_aos = compute_aos_flag_columns(gt, dt)
    if compute_aos and 'bbox' not in eval_types:
        raise ValueError('the alphas are valid, so kitti_eval computes AOS, which needs the bbox '
                         'metric: the reference fails on these eval_types')
    return _evaluate_packed(packed, classes, eval_types, compute_aos, return_intermediates,
                            overlap_limit)


def _evaluate_packed(packed, classes, eval_types, compute_aos, return_intermediates,
                     overlap_limit=None):
    if compute_aos and 'aos' not in eval_types:
        eval_types.append('aos')
    metrics = [m for m, n in enumerate(METRICS) if n in eval_types]
    ev = KittiEvaluator(classes, metrics, 'aos' in eval_types, overlap_limit)
    try:
        pr, cnt = ev.forward(packed)
    finally:
        ev.close()
    per = len(classes) * 6
    rets = {}
    for ms, m in enumerate(metrics):
        rets[m] = precision_recall(pr[ms * per:(ms + 1) * per], cnt[ms * per:(ms + 1) * per],
                                   len(classes), m == 0 and 'aos' in eval_types)
    result, ret_dict = report(classes, eval_types, compute_aos, rets)
    if return_intermediates:
        return result, ret_dict, {'pr': pr, 'thr_count': cnt, 'rets': rets}
    return result, ret_dict


# ---------------------------------------------------------------------------------------------
# KittiDataset.format_results / bbox2result_kitti / evaluate (mmdet3d datasets/kitti_dataset.py)
# restated on CPU float32 tensors with the same torch / numpy operations as the reference's
# LiDARInstance3DBoxes.limit_yaw / convert_to / CameraInstance3DBoxes.corners / points_cam2img.

KITTI_PCD_LIMIT_RANGE = (0, -40, -3, 70.4, 40, 0.0)


def _limit_period(val, offset=0.5, period=np.pi):
    import torch
    return val - torch.floor(val / period + offset) * period


def _lidar_to_cam(t, rt_mat):
    """Box3DMode.convert(LIDAR -> CAM) of a [K, 7] float32 tensor."""
    import torch
    x_size, y_size, z_size = t[..., 3:4], t[..., 4:5], t[..., 5:6]
    yaw = t[..., 6:7]
    if rt_mat is None:
        rt_mat = t.new_tensor([[0, -1, 0], [0, 0, -1], [1, 0, 0]])
    xyz_size = torch.cat([x_size, z_size, y_size], dim=-1)
    yaw = -yaw - np.pi / 2
    yaw = _limit_period(yaw, period=np.pi * 2)
    if not isinstance(rt_mat, torch.Tensor):
        rt_mat = t.new_tensor(rt_mat)
    if rt_mat.size(1) == 4:
        extended_xyz = torch.cat([t[..., :3], t.new_ones(t.size(0), 1)], dim=-1)
        xyz = extended_xyz @ rt_mat.t()
    else:
        xyz = t[..., :3] @ rt_mat.t()
    return torch.cat([xyz[..., :3], xyz_size, yaw], dim=-1)


def _cam_corners(cam):
    """CameraInstance3DBoxes.corners: [K, 8, 3]."""
    import torch
    dims = cam[:, 3:6]
    corners_norm = torch.from_numpy(np.stack(np.unravel_index(np.arange(8), [2] * 3),
                                             axis=1)).to(device=dims.device, dtype=dims.dtype)
    corners_norm = corners_norm[[0, 1, 3, 2, 4, 5, 7, 6]]
    corners_norm = corners_norm - dims.new_tensor([0.5, 1, 0.5])
    corners = dims.view([-1, 1, 3]) * corners_norm.reshape([1, 8, 3])
    angles = cam[:, 6]
    rot_sin, rot_cos = torch.sin(angles), torch.cos(angles)
    ones, zeros = torch.ones_like(rot_cos), torch.zeros_like(rot_cos)
    rot_mat_T = torch.stack([torch.stack([rot_cos, zeros, -rot_sin]),
                             torch.stack([zeros, ones, zeros]),
                             torch.stack([rot_sin, zeros, rot_cos])])
    corners = torch.einsum('aij,jka->aik', corners, rot_mat_T)
    corners += cam[:, :3].view(-1, 1, 3)
    return corners


def _points_cam2img(points_3d, proj_mat):
    import torch
    shape = list(points_3d.shape)
    shape[-1] = 1
    d1, d2 = proj_mat.shape[:2]
    if not ((d1 == 3 and d2 in (3, 4)) or (d1 == 4 and d2 == 4)):
        raise ValueError(f'P2 of shape {tuple(proj_mat.shape)} is not 3x3, 3x4 or 4x4')
    if d1 == 3:
        expanded = torch.eye(4, device=proj_mat.device, dtype=proj_mat.dtype)
        expanded[:d1, :d2] = proj_mat
        proj_mat = expanded
    points_4 = torch.cat([points_3d, points_3d.new_ones(shape)], dim=-1)
    point_2d = points_4 @ proj_mat.T
    return point_2d[..., :2] / point_2d[..., 2:3]


def _boxes_tensor(boxes):
    import torch
    t = boxes.tensor if hasattr(boxes, 'tensor') else boxes
    t = torch.as_tensor(t, dtype=torch.float32).detach().cpu()
    if t.numel() == 0:
        t = t.reshape(0, 7)
    if t.dim() != 2 or t.size(-1) < 7:
        raise ValueError(f'boxes_3d must be [K, >=7], got {tuple(t.shape)}')
    return t[:, :7].clone()


def convert_valid_bboxes(box_dict, info, pcd_limit_range=KITTI_PCD_LIMIT_RANGE,
                         pseudo_lidar=False):
    """KittiDataset.convert_valid_bboxes: LiDAR boxes -> 2-D boxes, camera and LiDAR boxes of
    the ones inside the image and the range.  ``boxes_3d`` is a [K, 7] tensor (or a box
    structure with ``.tensor``) in LiDAR coordinates, bottom centre."""
    import torch
    t = _boxes_tensor(box_dict['boxes_3d'])
    scores = torch.as_tensor(box_dict['scores_3d']).detach().cpu()
    labels = torch.as_tensor(box_dict['labels_3d']).detach().cpu()
    if len(scores) != len(t) or len(labels) != len(t):
        raise ValueError('boxes_3d, scores_3d and labels_3d differ in length')
    sample_idx = info['image']['image_idx']
    t[:, 6] = _limit_period(t[:, 6], 0.5, np.pi * 2)
    empty = dict(bbox=np.zeros([0, 4]), box3d_camera=np.zeros([0, 7]),
                 box3d_lidar=np.zeros([0, 7]), scores=np.zeros([0]),
                 label_preds=np.zeros([0]), sample_idx=sample_idx)
    if len(t) == 0:
        return empty
    rect = info['calib']['R0_rect'].astype(np.float32)
    Trv2c = info['calib']['Tr_velo_to_cam'].astype(np.float32)
    P2 = t.new_tensor(info['calib']['P2'].astype(np.float32))
    img_shape = info['image']['image_shape']
    cam = _lidar_to_cam(t, None if pseudo_lidar else rect @ Trv2c)
    corners_img = _points_cam2img(_cam_corners(cam), P2)
    minxy = torch.min(corners_img, dim=1)[0]
    maxxy = torch.max(corners_img, dim=1)[0]
    box_2d = torch.cat([minxy, maxxy], dim=1)
    image_shape = t.new_tensor(img_shape)
    valid_cam = ((box_2d[:, 0] < image_shape[1]) & (box_2d[:, 1] < image_shape[0]) &
                 (box_2d[:, 2] > 0) & (box_2d[:, 3] > 0))
    limit_range = t.new_tensor(pcd_limit_range)
    center = t[:, :3]
    valid_pcd = (center > limit_range[:3]) & (center < limit_range[3:])
    valid = valid_cam & valid_pcd.all(-1)
    if valid.sum() > 0:
        return dict(bbox=box_2d[valid, :].numpy(), box3d_camera=cam[valid].numpy(),
                    box3d_lidar=t[valid].numpy(), scores=scores[valid].numpy(),
                    label_preds=labels[valid].numpy(), sample_idx=sample_idx)
    empty['label_preds'] = np.zeros([0, 4])
    return empty


def _unwrap_results(results):
    if len(results) == 0:
        raise ValueError('no results')
    if not isinstance(results[0], dict):
        raise ValueError('2-D-only results (bbox2result_kitti2d) are not supported')
    if 'img_bbox' in results[0]:
        raise ValueError("'img_bbox' results (bbox2result_kitti2d) are not supported")
    if 'pts_bbox' in results[0]:
        results = [r['pts_bbox'] for r in results]
    for r in results:
        missing = [k for k in ('boxes_3d', 'scores_3d', 'labels_3d') if k not in r]
        if missing:
            raise ValueError(f'a result lacks {missing}')
    return results


def bbox2result_kitti(results, data_infos, class_names,
                      pcd_limit_range=KITTI_PCD_LIMIT_RANGE, pseudo_lidar=False,
                      submission_prefix=None):
    """KittiDataset.bbox2result_kitti: per frame, the KITTI-format anno dict kitti_eval reads.
    With ``submission_prefix``, writes ``<prefix>/<image_idx:06d>.txt`` in the benchmark's
    format.  DfM's KITTI config sets ``pseudo_lidar=True``."""
    import os
    results = _unwrap_results(results)
    if len(results) != len(data_infos):
        raise ValueError(f'{len(results)} results but {len(data_infos)} data_infos')
    if submission_prefix is not None:
        os.makedirs(submission_prefix, exist_ok=True)
    det_annos = []
    for pred_dicts, info in zip(results, data_infos):
        sample_idx = info['image']['image_idx']
        image_shape = info['image']['image_shape'][:2]
        box_dict = convert_valid_bboxes(pred_dicts, info, pcd_limit_range, pseudo_lidar)
        anno = {k: [] for k in ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions',
                                'location', 'rotation_y', 'score')}
        if len(box_dict['bbox']) > 0:
            for box, box_lidar, bbox, score, label in zip(
                    box_dict['box3d_camera'], box_dict['box3d_lidar'], box_dict['bbox'],
                    box_dict['scores'], box_dict['label_preds']):
                if not 0 <= int(label) < len(class_names):
                    raise ValueError(f'label {int(label)} has no class name')
                bbox[2:] = np.minimum(bbox[2:], image_shape[::-1])
                bbox[:2] = np.maximum(bbox[:2], [0, 0])
                anno['name'].append(class_names[int(label)])
                anno['truncated'].append(0.0)
                anno['occluded'].append(0)
                anno['alpha'].append(-np.arctan2(-box_lidar[1], box_lidar[0]) + box[6])
                anno['bbox'].append(bbox)
                anno['dimensions'].append(box[3:6])
                anno['location'].append(box[:3])
                anno['rotation_y'].append(box[6])
                anno['score'].append(score)
            anno = {k: np.stack(v) for k, v in anno.items()}
        else:
            anno = {'name': np.array([]), 'truncated': np.array([]), 'occluded': np.array([]),
                    'alpha': np.array([]), 'bbox': np.zeros([0, 4]),
                    'dimensions': np.zeros([0, 3]), 'location': np.zeros([0, 3]),
                    'rotation_y': np.array([]), 'score': np.array([])}
        if submission_prefix is not None:
            with open(f'{submission_prefix}/{sample_idx:06d}.txt', 'w') as f:
                bbox, loc, dims = anno['bbox'], anno['location'], anno['dimensions']
                for i in range(len(bbox)):
                    print('{} -1 -1 {:.4f} {:.4f} {:.4f} {:.4f} '
                          '{:.4f} {:.4f} {:.4f} '
                          '{:.4f} {:.4f} {:.4f} {:.4f} {:.4f} {:.4f}'.format(
                              anno['name'][i], anno['alpha'][i], bbox[i][0], bbox[i][1],
                              bbox[i][2], bbox[i][3], dims[i][1], dims[i][2], dims[i][0],
                              loc[i][0], loc[i][1], loc[i][2], anno['rotation_y'][i],
                              anno['score'][i]), file=f)
        anno['sample_idx'] = np.array([sample_idx] * len(anno['score']), dtype=np.int64)
        det_annos.append(anno)
    return det_annos


def evaluate(results, data_infos, class_names, pcd_limit_range=KITTI_PCD_LIMIT_RANGE,
             pseudo_lidar=False, submission_prefix=None, return_str=False):
    """KittiDataset.evaluate for 3-D results: bbox2result_kitti, then kitti_eval against
    ``info['annos']``.  As in the reference, plain per-frame dicts (what ``DfM.simple_test``
    returns) give kitti_eval's ret_dict as it is; results wrapped as ``{'pts_bbox': ...}`` give
    ``pts_bbox/KITTI/...`` keys with each value rounded as ``float('{:.4f}'.format(ap))``.
    With ``return_str`` the report string comes second."""
    wrapped = len(results) > 0 and isinstance(results[0], dict) and 'pts_bbox' in results[0]
    dt_annos = bbox2result_kitti(results, data_infos, class_names, pcd_limit_range,
                                 pseudo_lidar, submission_prefix)
    gt_annos = [info['annos'] for info in data_infos]
    result_str, ap_dict = kitti_eval(gt_annos, dt_annos, list(class_names))
    if wrapped:
        ap_dict = {f'pts_bbox/{k}': float('{:.4f}'.format(v)) for k, v in ap_dict.items()}
    return (ap_dict, result_str) if return_str else ap_dict
