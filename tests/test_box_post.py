"""get_bboxes of both anchor heads (dense_heads/anchor3d_head.py:407-547, box3d_nms.py) on CUDA
(``dfm_box_post_*``, ``modules.{LIGAAnchor3DHead,Anchor3DHead}.get_bboxes``).

CPU: the torch restatement ``tests/box_post_oracle.py`` reproduces ``tests/golden/box_post.npz``
(written by the reference's own functions) bit for bit; the module's anchor tables equal the
reference generators'; the nms_rotated stand-in on hand-worked pairs; the descriptor ABI.
GPU: synthetic head outputs at the shipped grids and the real regressions of both all-CUDA
chains, fed to the library and to the restatement on the same GPU tensors."""
import ctypes
import hashlib
import math
import os
import subprocess
import shutil

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import synthetic as syn
from tests import box_post_oracle as BP
from tests.util import GOLDEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-5


def _golden():
    return np.load(os.path.join(GOLDEN, 'box_post.npz'))


def _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset, num_classes=3):
    with torch.no_grad():
        return BP.get_bboxes_single(cls, box, dirc, anchors, cfg, num_classes, sigmoid,
                                    dir_offset, 0.0)


# ---------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize('name', list(syn.BOX_POST_CASES))
def test_oracle_matches_reference_golden(name):
    generator, ny, nx, cfg, sigmoid, dir_offset, seed, kw = syn.BOX_POST_CASES[name]
    g = _golden()
    cls, box, dirc = syn.make_box_post_case(seed, ny, nx, **kw)
    assert sum(t.double().abs().sum().item() for t in (cls, box, dirc)) == \
        float(g[f'{name}.input_sum'])
    anchors = modules.grid_anchors(generator, ny, nx, 'cpu')
    assert torch.equal(anchors, torch.from_numpy(g[f'{name}.anchors']))
    r = _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset)
    assert torch.equal(r['boxes'], torch.from_numpy(g[f'{name}.boxes']))
    assert torch.equal(r['scores'], torch.from_numpy(g[f'{name}.scores']))
    assert torch.equal(r['labels'], torch.from_numpy(g[f'{name}.labels']))
    n_anchor = ny * nx * 6
    assert (r['topk'] is not None) == (n_anchor > cfg['nms_pre'])
    if name == 'kitti_max_num_empty_class':
        assert len(r['candidates'][2]) == 0 and len(r['boxes']) == cfg['max_num']
        assert sum(len(k) for k in r['keep']) > cfg['max_num']


@pytest.mark.parametrize('name,generator,ny,nx', [
    ('kitti', syn.KITTI_ANCHOR_GENERATOR, 304, 288), ('waymo', syn.WAYMO_ANCHOR_GENERATOR, 300, 220)])
def test_anchor_table_at_shipped_grid(name, generator, ny, nx):
    g = _golden()
    a = modules.grid_anchors(generator, ny, nx, 'cpu').contiguous()
    assert tuple(a.shape) == tuple(g[f'{name}_full.shape'])
    assert hashlib.sha256(a.numpy().tobytes()).hexdigest() == str(g[f'{name}_full.anchors_sha256'])


def _box(x, y, w, h, r):
    return torch.tensor([x, y, w, h, r], dtype=torch.float64)


def test_rotated_iou_hand_cases():
    """Identical boxes: 1.  Disjoint: 0.  A unit square at 45 degrees centred in a 2 x 2 square
    lies inside it: IoU = 1 / 4."""
    a = _box(3.0, -2.0, 4.0, 1.5, 0.7)
    assert float(BP.rotated_iou(a, a)) == pytest.approx(1.0, abs=1e-12)
    assert float(BP.rotated_iou(a, _box(30.0, 5.0, 4.0, 1.5, 0.7))) == 0.0
    assert float(BP.rotated_iou(_box(1, 1, 2, 2, 0.0), _box(1, 1, 1, 1, math.pi / 4))) == \
        pytest.approx(0.25, abs=1e-12)


def test_rotated_iou_corner_convention(monkeypatch):
    """Two 4 x 1 boxes at yaw pi/4, centres (0, 0) and (1, 1).  With mmcv's corners
    (centre + R(-yaw)(+-w/2, +-h/2)) the long axis runs along (1, -1)/sqrt 2: the centre offset
    (1, 1) is perpendicular to it at distance sqrt 2 > h = 1, so the boxes are disjoint, IoU 0,
    below nms_thr 0.25.  With R(+yaw) (LiDARInstance3DBoxes.corners) the long axis runs along
    the offset: overlap (4 - sqrt 2) x 1 = 2.586, union 8 - 2.586 = 5.414, IoU 0.4776 > 0.25."""
    a, b = _box(0, 0, 4, 1, math.pi / 4), _box(1, 1, 4, 1, math.pi / 4)
    assert BP.NMS_ROTATED_ROT_SIGN == -1.0
    assert float(BP.rotated_iou(a, b)) == 0.0
    monkeypatch.setattr(BP, 'NMS_ROTATED_ROT_SIGN', 1.0)
    s2 = math.sqrt(2)
    assert float(BP.rotated_iou(a, b)) == pytest.approx((4 - s2) / (4 + s2), abs=1e-12)


def test_kernel_states_the_same_convention():
    src = open(os.path.join(ROOT, 'depth_from_motion_b200', 'csrc', 'box_post_kernels.cuh')).read()
    assert 'constexpr float BP_ROT_SIGN = -1.f;' in src


@pytest.mark.skipif(shutil.which('gcc') is None, reason='no C compiler')
def test_box_post_desc_matches_the_c_header(tmp_path):
    cls = capi.BoxPostDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>',
             f'#include "{os.path.join(ROOT, "include", "dfm_b200.h")}"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(dfm_box_post_desc_t));']
    lines += [f'printf("{f} %zu\\n", offsetof(dfm_box_post_desc_t, {f}));' for f, _ in cls._fields_]
    lines += ['return 0;', '}']
    (tmp_path / 'abi.c').write_text('\n'.join(lines))
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-o', str(tmp_path / 'abi'),
                    str(tmp_path / 'abi.c')], check=True)
    got = dict(l.split() for l in subprocess.run([str(tmp_path / 'abi')], capture_output=True,
                                                 text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _kitti_head(**cfg):
    return modules.LIGAAnchor3DHead(
        num_classes=3, in_channels=64, feat_channels=64, norm_cfg=dict(type='GN', num_groups=32),
        anchor_generator=syn.KITTI_ANCHOR_GENERATOR, dir_offset=syn.KITTI_DIR_OFFSET,
        test_cfg=dict(syn.KITTI_TEST_CFG, **cfg))


def _waymo_head(sigmoid=True, **cfg):
    return modules.Anchor3DHead(
        num_classes=3, in_channels=256, anchor_generator=syn.WAYMO_ANCHOR_GENERATOR,
        dir_offset=syn.WAYMO_DIR_OFFSET, test_cfg=dict(syn.WAYMO_TEST_CFG, **cfg),
        loss_cls=dict(type='FocalLoss', use_sigmoid=sigmoid))


def test_unsupported_options_raise():
    cls, box, dirc = (t[None] for t in syn.make_box_post_case(1, 4, 4))
    with pytest.raises(NotImplementedError):
        _kitti_head(use_rotate_nms=False).get_bboxes([cls], [box], [dirc], [{}])
    with pytest.raises(NotImplementedError):
        _waymo_head().get_bboxes([cls], [box], None, [{}])
    with pytest.raises(NotImplementedError):
        _waymo_head().get_bboxes([cls], [box], [None], [{}])
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        _waymo_head().get_bboxes([cls], [box], [dirc], [{}])


# ---------------------------------------------------------------------------------- GPU

def _nms_validity(bev, cand, keep, thr):
    """fp64 IoU in processing order: a kept box overlaps no earlier kept box by more than
    thr + EPS; a suppressed one overlaps some earlier kept box by more than thr - EPS.  Returns
    the number of decisions within EPS of thr."""
    n = len(cand)
    if n == 0:
        return 0
    pos = {int(a): i for i, a in enumerate(cand.tolist())}
    kept = torch.zeros(n, dtype=torch.bool, device=bev.device)
    kept[[pos[int(a)] for a in keep.tolist()]] = True
    iou = BP.rotated_iou(bev[:, None], bev[kept][None])           # [n, kept]
    kidx = torch.nonzero(kept).flatten()
    earlier = kidx[None, :] < torch.arange(n, device=bev.device)[:, None]
    m = torch.where(earlier, iou, torch.full_like(iou, -1.0)).max(dim=1)[0]
    assert bool((m[kept] <= thr + EPS).all()), float(m[kept].max())
    assert bool((m[~kept] > thr - EPS).all()), float(m[~kept].min())
    return int(((m - thr).abs() <= EPS).sum())


def _check_against_oracle(head, cls, box, dirc, anchors, cfg, sigmoid, dir_offset, label):
    """One sample through head.get_bboxes and the oracle on the same GPU tensors."""
    (boxes, scores, labels), = head.get_bboxes([cls[None]], [box[None]], [dirc[None]], [{}])
    capi.sync_check()
    r = _oracle(cls, box, dirc, anchors, cfg, sigmoid, dir_offset)
    bp = head._box_post
    # top-k, tie-aware
    if r['topk'] is not None:
        got = bp.debug_tensor('topk_index')[0].long()
        ref = r['topk']
        ncol = 3 if sigmoid else 4
        sc = cls.permute(1, 2, 0).reshape(-1, ncol)
        sc = (sc.sigmoid() if sigmoid else sc.softmax(-1)[:, :-1]).max(1)[0]
        assert torch.equal(torch.sort(sc[got], descending=True)[0], sc[got]), 'not sorted'
        kth = sc[ref[-1]]
        diff_g = set(got.tolist()) - set(ref.tolist())
        diff_r = set(ref.tolist()) - set(got.tolist())
        assert all(float(sc[i]) == float(kth) for i in diff_g | diff_r), 'top-k differs off ties'
    # candidates and keeps per class
    ties_band = 0
    bev_all = None
    same_keep = True
    slot_anchor = r['topk'] if r['topk'] is not None else torch.arange(cls.shape[-1] *
                                                                       cls.shape[-2] * 6,
                                                                       device=cls.device)
    with torch.no_grad():
        dec = BP.decode(anchors[slot_anchor],
                        box.permute(1, 2, 0).reshape(-1, 7)[slot_anchor])
        bev_all = BP.nms_box(dec)
    slot_of = torch.full((anchors.shape[0],), -1, dtype=torch.long, device=cls.device)
    slot_of[slot_anchor] = torch.arange(len(slot_anchor), device=cls.device)
    for c in range(3):
        cand = bp.debug_tensor(f'cls{c}_candidates')[0].long()
        cand = cand[cand >= 0]
        keep = bp.debug_tensor(f'cls{c}_keep')[0].long()
        keep = keep[keep >= 0]
        assert set(cand.tolist()) == set(r['candidates'][c].tolist()), (label, c)
        band = _nms_validity(bev_all[slot_of[cand]], cand, keep, cfg['nms_thr'])
        ties_band += band
        if band == 0:
            assert torch.equal(keep, r['keep'][c]), (label, c)
        same_keep &= torch.equal(keep, r['keep'][c])
        print(label, 'class', c, 'candidates', len(cand), 'kept', len(keep), 'band', band)
    if same_keep:
        assert torch.equal(labels, r['labels'])
        assert torch.equal(scores, r['scores'])
        torch.testing.assert_close(boxes, r['boxes'], rtol=2.4e-7, atol=1e-6)
    return boxes, scores, labels, ties_band


@pytest.mark.gpu
@pytest.mark.parametrize('shape', ['kitti', 'waymo'])
def test_shipped_shape_vs_oracle(shape):
    if shape == 'kitti':
        ny, nx, head, gen = 304, 288, _kitti_head(), syn.KITTI_ANCHOR_GENERATOR
        cfg, dir_offset = syn.KITTI_TEST_CFG, syn.KITTI_DIR_OFFSET
    else:
        ny, nx, head, gen = 300, 220, _waymo_head(), syn.WAYMO_ANCHOR_GENERATOR
        cfg, dir_offset = syn.WAYMO_TEST_CFG, syn.WAYMO_DIR_OFFSET
    cls, box, dirc = (t.cuda() for t in syn.make_box_post_case(11, ny, nx))
    anchors = modules.grid_anchors(gen, ny, nx, 'cuda')
    l0, _ = capi.launch_counters()
    boxes, scores, labels, band = _check_against_oracle(head, cls, box, dirc, anchors, cfg, True,
                                                        dir_offset, shape)
    assert capi.launch_counters()[0] > l0
    assert 0 < len(boxes) <= cfg['max_num']
    print(shape, 'boxes', len(boxes), 'decisions within EPS of nms_thr', band)


@pytest.mark.gpu
def test_softmax_arm_vs_oracle():
    generator, ny, nx, cfg, sigmoid, dir_offset, seed, kw = syn.BOX_POST_CASES['waymo_softmax']
    cls, box, dirc = (t.cuda() for t in syn.make_box_post_case(seed, ny, nx, **kw))
    anchors = modules.grid_anchors(generator, ny, nx, 'cuda')
    head = _waymo_head(sigmoid=False, **{k: v for k, v in cfg.items()})
    # softmax: scores may differ from torch's by rounding; check the NMS and the set sizes
    (boxes, scores, labels), = head.get_bboxes([cls[None]], [box[None]], [dirc[None]], [{}])
    r = _oracle(cls, box, dirc, anchors, cfg, False, dir_offset)
    assert len(boxes) == len(r['boxes'])
    torch.testing.assert_close(scores, r['scores'], rtol=1e-6, atol=1e-7)


def _run(head, cls, box, dirc, metas):
    out = head.get_bboxes([cls], [box], [dirc], metas)
    capi.sync_check()
    return out


@pytest.mark.gpu
def test_repeatable_batched_and_empty():
    ny, nx = 300, 220
    cases = [syn.make_box_post_case(s, ny, nx) for s in (21, 22)]
    cls, box, dirc = (torch.stack([c[i] for c in cases]).cuda() for i in range(3))
    head = _waymo_head()
    a = _run(head, cls, box, dirc, [{}, {}])
    b = _run(head, cls, box, dirc, [{}, {}])
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    single = _waymo_head()
    for i in range(2):
        (bx, sc, lb), = _run(single, cls[i:i + 1], box[i:i + 1], dirc[i:i + 1], [{}])
        assert torch.equal(bx, a[i][0]) and torch.equal(sc, a[i][1]) and torch.equal(lb, a[i][2])
    # nothing passes score_thr
    (bx, sc, lb), = _run(_waymo_head(score_thr=0.9999), torch.full_like(cls[:1], -9.0), box[:1],
                         dirc[:1], [{}])
    assert bx.shape == (0, 7) and sc.shape == (0,) and lb.shape == (0,)


def _desc(**kw):
    d = dict(num_classes=3, num_anchors=6, ny=300, nx=220, batch=1, use_sigmoid=1, nms_pre=4096,
             max_num=500, score_thr=0.001, nms_thr=0.05, dir_offset=-0.7854,
             dir_limit_offset=0.0)
    d.update(kw)
    return capi.BoxPostDesc(*[d[f] for f, _ in capi.BoxPostDesc._fields_])


@pytest.mark.gpu
def test_c_api_canaries_and_errors():
    L = capi.lib()
    ny, nx = 300, 220
    anchors = modules.grid_anchors(syn.WAYMO_ANCHOR_GENERATOR, ny, nx, 'cpu').contiguous()
    hd = ctypes.c_void_p()
    for bad in (dict(nms_pre=0), dict(nms_pre=5000), dict(num_classes=0), dict(num_classes=17),
                dict(batch=0), dict(max_num=0), dict(use_sigmoid=2), dict(nms_thr=float('nan'))):
        assert L.dfm_box_post_create(ctypes.byref(_desc(**bad)), modules._ptr(anchors),
                                     ctypes.byref(hd)) == 1, bad
    assert L.dfm_box_post_create(ctypes.byref(_desc()), None, ctypes.byref(hd)) == 1
    capi.check(L.dfm_box_post_create(ctypes.byref(_desc(max_num=50)), modules._ptr(anchors),
                                     ctypes.byref(hd)), 'create')
    try:
        cls, box, dirc = (t[None].cuda() for t in syn.make_box_post_case(31, ny, nx))
        boxes = torch.full((1, 50, 7), 123.0, device='cuda')
        scores = torch.full((1, 50), 123.0, device='cuda')
        labels = torch.full((1, 50), 77, device='cuda', dtype=torch.int32)
        count = torch.full((1,), -1, device='cuda', dtype=torch.int32)
        p = modules._ptr
        s = modules._stream()
        assert L.dfm_box_post_forward(hd, p(cls), p(box), None, p(boxes), p(scores), p(labels),
                                      p(count), s) == 1
        out = torch.empty(4096, device='cuda', dtype=torch.int32)
        assert L.dfm_box_post_debug_tensor(hd, b'topk_index', p(out), 4096, s) == 3
        # a tiny max_num with many kept boxes: exactly max_num written
        capi.check(L.dfm_box_post_forward(hd, p(cls), p(box), p(dirc), p(boxes), p(scores),
                                          p(labels), p(count), s), 'forward')
        capi.sync_check()
        assert int(count[0]) == 50
        assert L.dfm_box_post_debug_tensor(hd, b'topk_index', p(out), 4095, s) == 1
        assert L.dfm_box_post_debug_tensor(hd, b'cls9_keep', p(out), 4096, s) == 1
        # a sample with few boxes: canaries past count stay
        boxes.fill_(123.0)
        scores.fill_(123.0)
        labels.fill_(77)
        cls2 = torch.full_like(cls, -9.0)
        cls2[0, 0, 100, 100] = 3.0
        capi.check(L.dfm_box_post_forward(hd, p(cls2), p(box), p(dirc), p(boxes), p(scores),
                                          p(labels), p(count), s), 'forward')
        capi.sync_check()
        k = int(count[0])
        assert 1 <= k < 50
        assert bool((boxes[0, k:] == 123.0).all()) and bool((scores[0, k:] == 123.0).all())
        assert bool((labels[0, k:] == 77).all())
    finally:
        L.dfm_box_post_destroy(hd)


# Designed grids through the C entry point: one anchor per cell on a 1 x N grid, an anchor table
# of chosen boxes and zero box deltas, so the decoded boxes are the anchors and the exact IoU of
# every pair is known.

def _c_run(anchors, cls, C=1, nms_thr=0.25, max_num=4096, nms_pre=4096, sigmoid=1, dirc=None,
           dir_offset=0.0, dir_limit_offset=0.0):
    """dfm_box_post_forward on cls [B, ncol, 1, N] (zero box deltas, dirc [B, 2, 1, N] or zero
    direction logits); returns the outputs per sample with the candidate / keep lists per
    (sample, class) and 'topk' when the grid takes the top-k."""
    L, p, s = capi.lib(), modules._ptr, modules._stream()
    B, N = cls.shape[0], anchors.shape[0]
    reg = torch.zeros((B, 7, 1, N), device='cuda')
    if dirc is None:
        dirc = torch.zeros((B, 2, 1, N), device='cuda')
    desc = _desc(num_classes=C, num_anchors=1, ny=1, nx=N, batch=B, use_sigmoid=sigmoid,
                 nms_pre=nms_pre, max_num=max_num, score_thr=0.1, nms_thr=nms_thr,
                 dir_offset=dir_offset, dir_limit_offset=dir_limit_offset)
    hd = ctypes.c_void_p()
    host_anchors = anchors.cpu().contiguous()     # alive until create has copied it
    capi.check(L.dfm_box_post_create(ctypes.byref(desc), p(host_anchors), ctypes.byref(hd)),
               'create')
    try:
        boxes = torch.empty((B, max_num, 7), device='cuda')
        scores = torch.empty((B, max_num), device='cuda')
        labels = torch.empty((B, max_num), device='cuda', dtype=torch.int32)
        count = torch.empty((B,), device='cuda', dtype=torch.int32)
        capi.check(L.dfm_box_post_forward(hd, p(cls), p(reg), p(dirc), p(boxes), p(scores),
                                          p(labels), p(count), s), 'forward')
        K = min(N, nms_pre)
        names = [(c, kind) for c in range(C) for kind in ('candidates', 'keep')]
        names += ['topk'] if N > nms_pre else []
        dbg = {}
        for key in names:
            t = torch.empty((B, K), device='cuda', dtype=torch.int32)
            name = 'topk_index' if key == 'topk' else f'cls{key[0]}_{key[1]}'
            capi.check(L.dfm_box_post_debug_tensor(hd, name.encode(), p(t), t.numel(), s),
                       'debug')
            dbg[key] = t
        capi.sync_check()
    finally:
        L.dfm_box_post_destroy(hd)
    out = []
    for b in range(B):
        k = int(count[b])
        st = {key: v[b][v[b] >= 0].long() for key, v in dbg.items()}
        out.append((boxes[b, :k], scores[b, :k], labels[b, :k].long(), st))
    return out, reg, dirc


def _c_vs_oracle(anchors, cls, C=1, nms_thr=0.25, sigmoid=True, exact_scores=True, **kw):
    """Every sample's top-k and candidates equal the restatement's; so do its keep lists and
    outputs unless a decision lies within EPS of nms_thr, where both keep lists must be valid
    greedy NMS.  Softmax scores (exact_scores=False) may differ from torch's in the last bit.
    Returns the C results and the number of such decisions."""
    res, reg, dirc = _c_run(anchors, cls, C, nms_thr, sigmoid=int(sigmoid), **kw)
    cfg = dict(nms_pre=kw.get('nms_pre', 4096), score_thr=0.1, nms_thr=nms_thr,
               max_num=kw.get('max_num', 4096))
    with torch.no_grad():
        bev = BP.nms_box(BP.decode(anchors, torch.zeros_like(anchors)))
    band = 0
    for b, (boxes, scores, labels, st) in enumerate(res):
        with torch.no_grad():
            r = BP.get_bboxes_single(cls[b], reg[b], dirc[b], anchors, cfg, C, sigmoid,
                                     kw.get('dir_offset', 0.0), kw.get('dir_limit_offset', 0.0))
        if 'topk' in st:
            assert torch.equal(st['topk'], r['topk']), b
        same = True
        for c in range(C):
            cand, keep = st[c, 'candidates'], st[c, 'keep']
            assert torch.equal(cand, r['candidates'][c]), (b, c)
            near = _nms_validity(bev[cand], cand, keep, nms_thr)
            band += near
            if near == 0:
                assert torch.equal(keep, r['keep'][c]), (b, c, len(keep), len(r['keep'][c]))
            same &= torch.equal(keep, r['keep'][c])
        if same:
            assert torch.equal(labels, r['labels'])
            if exact_scores:
                assert torch.equal(scores, r['scores'])
            else:
                torch.testing.assert_close(scores, r['scores'], rtol=1e-6, atol=1e-7)
            bad = torch.nonzero(~torch.isclose(boxes, r['boxes'], rtol=2.4e-7,
                                               atol=1e-6).all(1)).flatten()
            assert len(bad) == 0, (bad[:4].tolist(), boxes[bad[:4]].tolist(),
                                   r['boxes'][bad[:4]].tolist())
    return res, band


def _along(yaw, du, dv):
    """(du, dv) in a box's (w, h) axes under the NMS corner convention, as an (x, y) offset."""
    c, s = math.cos(yaw), BP.NMS_ROTATED_ROT_SIGN * math.sin(yaw)
    return du * c - dv * s, du * s + dv * c


_ULP_STEPS = np.array([(i, j) for i in range(-8, 9) for j in range(-8, 9)], dtype=np.int32)


def _collinear_grid(thr):
    """Anchors [N, 7] and logits [N] of equal boxes offset along their own axis, so their long or
    short edges lie on one line: pairs with exact IoU (side - s) / (side + s) between 0.0002
    and 0.005 below or above nms_thr, and greedy chains A, B, C with IoU(A, B), IoU(B, C) above
    nms_thr and IoU(A, C) below it (A suppresses B, so C is kept).  Each later box takes,
    among the fp32 centres within 8 ulp of its offset, the one whose NMS box lies closest to
    the first box's axis: the edges are collinear to within the corners' rounding.  900 groups 14 m apart, out
    to 203 m; groups[g] lists each group's rows."""
    rng = np.random.RandomState(int(thr * 100))
    rows, logits, groups = [], [], []
    gx = np.linspace(-203.0, 203.0, 30)
    centres = [(x, y) for x in gx for y in gx]
    rng.shuffle(centres)
    for g, (x0, y0) in enumerate(centres):
        yaw = float(rng.choice([0.0, math.pi / 2, math.pi / 4, -math.pi / 2]) if g % 4 == 0
                    else rng.uniform(-6.0, 6.0))
        w, l = rng.uniform(1.5, 2.2), rng.uniform(3.5, 5.0)
        axis = rng.randint(2)
        side = (w, l)[axis]
        if g % 5 == 4:   # chain: step with IoU thr + 0.1 twice, two steps apart fall below thr
            t = thr + 0.1
            steps = (0.0, 1.0, 2.0)
        else:
            t = thr + rng.choice([-1.0, 1.0]) * rng.uniform(0.0002, 0.005)
            steps = (0.0, 1.0)
        sft = side * (1 - t) / (1 + t)
        groups.append(list(range(len(rows), len(rows) + len(steps))))
        ux, uy = _along(yaw, 1.0, 0.0) if axis == 0 else _along(yaw, 0.0, 1.0)
        for k, m in enumerate(steps):
            row = np.array([x0 + m * sft * ux, y0 + m * sft * uy, -1.0, w, l, 1.6, yaw],
                           dtype=np.float32)
            if k > 0:    # the fp32 centre whose NMS box lies closest to the first box's axis
                cand = np.repeat(row[None], len(_ULP_STEPS), 0)
                cand[:, :2] = (row[:2].view(np.int32) + _ULP_STEPS).view(np.float32)
                bev = BP.nms_box(torch.from_numpy(cand)).double().numpy()
                first = BP.nms_box(torch.from_numpy(np.array(rows[groups[-1][0]],
                                                             dtype=np.float32)[None]))
                d = bev[:, :2] - first.double().numpy()[:, :2]
                row = cand[np.argmin(np.abs(d[:, 0] * uy - d[:, 1] * ux))]
            rows.append(tuple(row.tolist()))
            logits.append(3.0 - 0.5 * k - 1e-3 * g)
    return (torch.tensor(rows, dtype=torch.float32), torch.tensor(logits, dtype=torch.float32),
            groups)


@pytest.mark.skipif(shutil.which('g++') is None, reason='no C++ compiler')
@pytest.mark.parametrize('thr', [0.05, 0.25])
def test_collinear_grid_flips_the_edge_clipping_iou(thr, tmp_path):
    """The collinear grid below is one an fp32 edge-clipping (Green's theorem) IoU gets wrong:
    on its NMS boxes (after the fp32 round trip) that IoU decides some pair the other way from
    the exact IoU, so the GPU test can tell the two forms apart."""
    from tests import test_rotated_iou as R
    anchors, _, groups = _collinear_grid(thr)
    bev = BP.nms_box(BP.decode(anchors, torch.zeros_like(anchors))).numpy()
    pairs = [(g[0], g[1]) for g in groups if len(g) == 2]
    a = np.ascontiguousarray(bev[[i for i, _ in pairs]])
    b = np.ascontiguousarray(bev[[j for _, j in pairs]])
    old = R.green_iou(a, b, tmp_path)
    ex = np.array([R.exact_iou(x, y) for x, y in zip(a, b)])
    assert bool((np.abs(ex - thr) >= 1.5e-4).all())
    flips = int(((old > thr) != (ex > thr)).sum())
    print('pairs', len(pairs), 'decisions flipped by the edge-clipping IoU', flips)
    assert flips >= 2


@pytest.mark.gpu
@pytest.mark.parametrize('thr', [0.05, 0.25])
def test_collinear_duplicates_and_chains_vs_oracle(thr):
    """The collinear grid through dfm_box_post_*: the keep lists must equal the
    restatement's, with no decision within EPS of nms_thr."""
    anchors, logits, groups = _collinear_grid(thr)
    anchors, cls = anchors.cuda(), logits.cuda().view(1, 1, 1, -1)
    ((_, _, _, st),), band = _c_vs_oracle(anchors, cls, nms_thr=thr)
    assert band == 0
    assert len(groups) < len(st[0, 'keep']) < len(anchors)


@pytest.mark.gpu
@pytest.mark.parametrize('n,nms_pre', [(300, 100), (101, 100), (100, 100)])
def test_topk_ties_take_the_lowest_anchors(n, nms_pre):
    """All logits equal: the top-k is the first nms_pre anchors by index (N = nms_pre + 1 drops
    the last one; N = nms_pre takes no top-k at all)."""
    rng = np.random.RandomState(n)
    a = np.stack([rng.uniform(-60, 60, n), rng.uniform(-60, 60, n), np.full(n, -1.0),
                  rng.uniform(1.5, 2.2, n), rng.uniform(3.5, 5.0, n), np.full(n, 1.6),
                  rng.uniform(-math.pi, math.pi, n)], 1)
    anchors = torch.tensor(a, dtype=torch.float32, device='cuda')
    cls = torch.full((1, 1, 1, n), 1.5, device='cuda')
    ((_, _, _, st),), _ = _c_vs_oracle(anchors, cls, nms_pre=nms_pre, max_num=500)
    assert ('topk' in st) == (n > nms_pre)
    if n > nms_pre:
        assert torch.equal(st['topk'], torch.arange(nms_pre, device='cuda'))
    assert torch.equal(st[0, 'candidates'], torch.arange(min(n, nms_pre), device='cuda'))


@pytest.mark.gpu
@pytest.mark.parametrize('sigmoid', [True, False])
def test_sixteen_classes_vs_oracle(sigmoid):
    """num_classes = 16 with sigmoid (16 columns) and with softmax (ncol = 17, background last)
    on a crowded grid with top-k."""
    rng = np.random.RandomState(16 + sigmoid)
    n, C = 200, 16
    a = np.stack([rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), np.full(n, -1.0),
                  rng.uniform(1.5, 2.2, n), rng.uniform(3.5, 5.0, n), np.full(n, 1.6),
                  rng.uniform(-math.pi, math.pi, n)], 1)
    anchors = torch.tensor(a, dtype=torch.float32, device='cuda')
    ncol = C if sigmoid else C + 1
    logits = rng.uniform(-4.0, 4.0, (ncol, n))
    if not sigmoid:
        logits[C] -= 2.0       # background: leave foreground scores above score_thr
    cls = torch.tensor(logits, dtype=torch.float32, device='cuda').view(1, ncol, 1, n)
    ((_, _, labels, st),), band = _c_vs_oracle(anchors, cls, C=C, sigmoid=sigmoid,
                                               exact_scores=sigmoid, nms_pre=150, max_num=1000)
    assert 'topk' in st
    assert len(set(labels.tolist())) == C
    print('sigmoid' if sigmoid else 'softmax', 'boxes', len(labels), 'band', band)


@pytest.mark.gpu
def test_max_num_cut_through_scores_equal_across_classes():
    """Three classes with bit-equal scores on runs of anchors (the same logit in every class
    column): the cut at max_num falls inside such a run, and the tie order (score descending,
    then class, then keep rank) must equal the restatement's stable sort of the class-major
    list."""
    n, C = 120, 3
    gx = np.arange(n) * 8.0 - 480.0           # 8 m apart: every box is kept in every class
    a = np.stack([gx, np.zeros(n), np.full(n, -1.0), np.full(n, 1.8), np.full(n, 4.0),
                  np.full(n, 1.6), np.zeros(n)], 1)
    anchors = torch.tensor(a, dtype=torch.float32, device='cuda')
    base = np.repeat(np.linspace(3.0, 1.0, 12), 10)          # runs of 10 equal logits
    cls = torch.tensor(np.stack([base] * C), dtype=torch.float32,
                       device='cuda').view(1, C, 1, n)
    for max_num in (45, 95, 200):                             # 45, 95: inside a run of ties
        ((_, scores, labels, st),), _ = _c_vs_oracle(anchors, cls, C=C, max_num=max_num)
        assert len(labels) == min(max_num, n * C)
        assert len(st[0, 'keep']) == n
    assert int((scores == scores[0]).sum()) == C * 10


@pytest.mark.gpu
def test_yaw_fix_at_period_boundaries():
    """Decoded yaws within a few ulp of dir_offset + k pi, where (yaw - dir_offset) / pi +
    dir_limit_offset is within about one ulp of an integer, with both direction labels: the
    boxes equal those of the restatement run on the CPU bit for bit (the kernel's yaw fix
    divides by pi as torch's CPU path does)."""
    off = syn.KITTI_DIR_OFFSET
    yaws = []
    for k in np.arange(-3.0, 3.5, 0.5):     # boundaries of dir_limit_offset 0 / 1 and 0.5
        y = np.float32(off + k * math.pi)
        for d in range(-3, 4):
            yaws.append((y.view(np.int32) + d).view(np.float32) if y != 0 else y)
    n = len(yaws)
    a = np.stack([np.arange(n) * 8.0 - 4.0 * n, np.zeros(n), np.full(n, -1.0),
                  np.full(n, 1.8), np.full(n, 4.0), np.full(n, 1.6), np.array(yaws)], 1)
    anchors = torch.tensor(a, dtype=torch.float32)
    logits = torch.linspace(3.0, 1.0, n).view(1, 1, 1, n)    # well apart: same order anywhere
    dirc = torch.zeros((1, 2, 1, n))
    dirc[0, 1, 0, 1::2] = 1.0                                  # label 1 on odd anchors
    for limit in (0.0, 0.5, 1.0):
        (got,), reg, _ = _c_run(anchors.cuda(), logits.cuda(), dirc=dirc.cuda(),
                                dir_offset=off, dir_limit_offset=limit, max_num=500)
        cfg = dict(nms_pre=4096, score_thr=0.1, nms_thr=0.25, max_num=500)
        with torch.no_grad():
            r = BP.get_bboxes_single(logits[0], reg[0].cpu(), dirc[0], anchors, cfg, 1, True,
                                     off, limit)
        assert torch.equal(got[2].cpu(), r['labels'])
        assert torch.equal(got[0].cpu(), r['boxes']), (limit, (got[0].cpu() - r['boxes'])
                                                       .abs().max(0)[0].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 63, 64, 65, 127, 128, 4095, 4096])
def test_candidate_counts_vs_oracle(n):
    """n candidates of one class in a crowded 40 m square: the diagonal IoU tile, the row and
    column blocks of the mask and the later words of the greedy sweep at the block edges.  Half
    the anchors score below score_thr."""
    rng = np.random.RandomState(n)
    N = 2 * n
    side = 40.0 * math.sqrt(N / 8192)
    a = np.stack([rng.uniform(-side, side, N), rng.uniform(-side, side, N), np.full(N, -1.0),
                  rng.uniform(1.5, 2.2, N), rng.uniform(3.5, 5.0, N), np.full(N, 1.6),
                  rng.uniform(-math.pi, math.pi, N)], 1)
    logits = rng.uniform(-1.0, 4.0, N)
    logits[rng.permutation(N)[:n]] = -5.0
    anchors = torch.tensor(a, dtype=torch.float32, device='cuda')
    cls = torch.tensor(logits, dtype=torch.float32, device='cuda').view(1, 1, 1, -1)
    ((_, _, _, st),), band = _c_vs_oracle(anchors, cls, nms_thr=0.25, nms_pre=min(N, 4096),
                                          max_num=4096)
    assert len(st[0, 'candidates']) == n
    print('candidates', n, 'kept', len(st[0, 'keep']), 'decisions within EPS of nms_thr', band)


@pytest.mark.gpu
def test_batch_with_an_empty_sample_equals_single_samples():
    """B = 2: sample 0 has no candidate, sample 1 has 4096; each equals its B = 1 run."""
    rng = np.random.RandomState(5)
    N = 4096
    a = np.stack([rng.uniform(-40, 40, N), rng.uniform(-40, 40, N), np.full(N, -1.0),
                  rng.uniform(1.5, 2.2, N), rng.uniform(3.5, 5.0, N), np.full(N, 1.6),
                  rng.uniform(-math.pi, math.pi, N)], 1)
    anchors = torch.tensor(a, dtype=torch.float32, device='cuda')
    cls = torch.stack([torch.full((1, 1, N), -5.0),
                       torch.tensor(rng.uniform(-1.0, 4.0, N), dtype=torch.float32)
                       .view(1, 1, N)]).cuda()
    both, _, _ = _c_run(anchors, cls, max_num=500)
    assert len(both[0][0]) == 0 and len(both[1][3][0, 'candidates']) == N
    for b in range(2):
        (one,), _, _ = _c_run(anchors, cls[b:b + 1].contiguous(), max_num=500)
        for u, v in zip(both[b][:3], one[:3]):
            assert torch.equal(u, v)
        for key in one[3]:
            assert torch.equal(both[b][3][key], one[3][key])
    _c_vs_oracle(anchors, cls[1:2].contiguous(), max_num=500)


@pytest.mark.gpu
def test_kitti_chain_end_to_end():
    """The real regressions of test_box_regression_parity_end_to_end's all-CUDA KITTI chain
    (DfMBackbone -> FrustumToVoxel -> BEVHourglass -> LIGAAnchor3DHead) through get_bboxes."""
    import copy

    from oracle import dfm_oracle as O
    from tests.test_gpu_parity import _backbone, _bev_modules, _frustum_module
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(23, h, w, d)
    cfg = syn.depth_cfg_for(d)
    fc = syn.make_frustum_case(24, h, w, d, (32, 28, 20))
    metas = copy.deepcopy(metas)
    metas[0]['cam2img'] = fc['metas'][0]['cam2img']
    bc = syn.make_bev_case(seed=25, nz=5, ny=28, nx=32)
    bb, fr = _backbone(params, cfg, 'auto'), _frustum_module(fc)
    bev, head = _bev_modules(bc)
    with torch.no_grad():
        cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        vol = fr(stereo, modules.CostLogits(cost, depth_samples=O.depth_samples(cfg)), metas,
                 fc['sem'].cuda())
        _, nz, ny, nx = vol.shape[1:]
        _, feat = bev(vol.view(1, -1, ny, nx))
        cls, box, dirc = head([feat])
    head.extra_cfg['anchor_generator'] = syn.KITTI_ANCHOR_GENERATOR
    head.extra_cfg['dir_offset'] = syn.KITTI_DIR_OFFSET
    cfg = dict(syn.KITTI_TEST_CFG, score_thr=0.3)
    head.test_cfg = cfg
    anchors = modules.grid_anchors(syn.KITTI_ANCHOR_GENERATOR, ny, nx, 'cuda')
    _check_against_oracle(head, cls[0][0], box[0][0], dirc[0][0], anchors, cfg, True,
                          syn.KITTI_DIR_OFFSET, 'kitti chain')


@pytest.mark.gpu
def test_waymo_chain_end_to_end():
    """lifting -> DfMNeck -> Anchor3DHead (the chain of test_waymo_box_regressions_end_to_end)
    through get_bboxes, two samples in one call checked one by one."""
    from tests.test_anchor3d_head import _cuda_head, load_fixture
    torch.backends.cudnn.allow_tf32 = False
    nv, t = 3, 2
    n_voxels, vrange = [20, 18, 12], [0.0, -9.0, -2.0, 20.0, 9.0, 4.0]
    rng = np.random.RandomState(61)
    mod = modules.DfMNeck(64, 256, num_frames=2)
    mod.load_state_dict(syn.make_neck_params(rng, mod.state_dict()), strict=True)
    mod = mod.cuda().eval()
    _, hp = load_fixture()
    head = _cuda_head(hp)

    class Host(modules.MultiViewDfMFeatureTransformation):
        pass
    host = Host()
    host.n_voxels, host.voxel_range = n_voxels, vrange
    host.temporal_aggregate, host.valid_sample, host.neck_3d = 'concat', True, mod
    feats, metas = [], []
    for b in range(2):
        f, m = syn.make_waymo_sample(70 + b, t, nv, feat_hw=(40, 64), input_hw=(160, 256),
                                     flip=bool(b), scale=1.0 + 0.02 * b, crop=(1.0 * b, 2.0 * b))
        k = np.array([[120., 0, 128, 0], [0, 120., 80, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        kfull = np.array([[1335.75, 0, 624, 0], [0, 1335.75, 416, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        m['ori_lidar2img'] = np.array([k @ np.linalg.inv(kfull) @ x
                                       for x in syn.waymo_lidar2img(t, nv)])
        feats.append(f)
        metas.append(m)
    with torch.no_grad():
        bev = host.feature_transformation(torch.stack(feats).cuda(), metas, nv, t)[0]
        cls, box, dirc = head([bev])
    head.extra_cfg['anchor_generator'] = syn.WAYMO_ANCHOR_GENERATOR
    head.dir_offset = syn.WAYMO_DIR_OFFSET
    head.test_cfg = syn.WAYMO_TEST_CFG
    ny, nx = cls[0].shape[-2:]
    anchors = modules.grid_anchors(syn.WAYMO_ANCHOR_GENERATOR, ny, nx, 'cuda')
    both = head.get_bboxes(cls, box, dirc, [{}, {}])
    capi.sync_check()
    for b in range(2):
        got = _check_against_oracle(head, cls[0][b], box[0][b], dirc[0][b], anchors,
                                    syn.WAYMO_TEST_CFG, True, syn.WAYMO_DIR_OFFSET,
                                    f'waymo chain {b}')
        for u, v in zip(both[b], got[:3]):
            assert torch.equal(u, v)
