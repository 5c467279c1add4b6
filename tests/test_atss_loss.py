"""DfM's 2-D auxiliary loss (``LIGAATSSHead.loss``).

CPU: the restatement's mmdet / mmcv stand-ins against hand-worked values and ``gradcheck`` in
fp64, the head's constructor and refusals.  GPU: the native targets, loss values and gradients
against the restatement (tests/atss_loss_oracle.py) at the shipped config and the 320 x 1280
training shape, on synthetic outputs and on the head's own forward, and at the assigner's and the
losses' decision edges."""
import math

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import modules
from depth_from_motion_b200 import synthetic as syn
from tests import anchor_loss_oracle as AO
from tests import atss_loss_oracle as O

STDS = syn.KITTI_ATSS_HEAD['bbox_coder']['target_stds']


# ---- CPU: the stand-ins ----

def test_delta_coder_round_trip_and_clamp():
    a = torch.tensor([[-32.0, -32.0, 32.0, 32.0], [0.0, 8.0, 16.0, 40.0]], dtype=torch.float64)
    g = torch.tensor([[-10.0, -20.0, 50.0, 30.0], [2.0, 6.0, 30.0, 33.0]], dtype=torch.float64)
    d = O.encode(a, g, STDS)
    # hand-worked: anchor 0 centre (0, 0) size 64; GT centre (20, 5) size (60, 50)
    assert d[0].tolist() == pytest.approx([20 / 64 / 0.1, 5 / 64 / 0.1, math.log(60 / 64) / 0.2,
                                           math.log(50 / 64) / 0.2], rel=1e-12)
    assert torch.allclose(O.decode(a, d, STDS), g, rtol=0, atol=1e-12)
    # size deltas clamp at |log(16 / 1000)|
    big = torch.tensor([[0.0, 0.0, 100.0, -100.0]], dtype=torch.float64)
    box = O.decode(a[:1], big, STDS)
    r = abs(math.log(16 / 1000))
    assert (box[0, 2] - box[0, 0]).item() == pytest.approx(64 * math.exp(r), rel=1e-12)
    assert (box[0, 3] - box[0, 1]).item() == pytest.approx(64 * math.exp(-r), rel=1e-12)


def test_giou_of_identical_nested_and_disjoint_boxes():
    b = torch.tensor([[0.0, 0.0, 4.0, 2.0]], dtype=torch.float64)
    assert O.giou_aligned(b, b).item() == pytest.approx(1.0, abs=1e-12)
    inner = torch.tensor([[1.0, 0.5, 3.0, 1.5]], dtype=torch.float64)
    assert O.giou_aligned(inner, b).item() == pytest.approx(2 / 8, rel=1e-9)
    # disjoint: IoU 0, enclosure 10 x 2 = 20, union 16: 0 - (20 - 16) / 20
    far = torch.tensor([[6.0, 0.0, 10.0, 2.0]], dtype=torch.float64)
    assert O.giou_aligned(b, far).item() == pytest.approx(-0.2, rel=1e-9)


def test_bce_and_focal_match_hand_values():
    x = torch.tensor([0.0, 2.0], dtype=torch.float64)
    t = torch.tensor([0.5, 0.25], dtype=torch.float64)
    got = torch.nn.functional.binary_cross_entropy_with_logits(x, t, reduction='none')
    want = [-(0.5 * math.log(0.5) + 0.5 * math.log(0.5)),
            -(0.25 * math.log(1 / (1 + math.exp(-2))) + 0.75 * math.log(1 - 1 / (1 + math.exp(-2))))]
    assert got.tolist() == pytest.approx(want, rel=1e-12)
    f = AO.sigmoid_focal_loss(torch.tensor([[0.0, 0.0]], dtype=torch.float64), torch.tensor([1]))
    # not the target: -(1 - a) p^2 log(1 - p); the target: -a (1 - p)^2 log p; p = 1/2
    assert f[0].tolist() == pytest.approx([-0.75 * 0.25 * math.log(0.5),
                                           -0.25 * 0.25 * math.log(0.5)], rel=1e-12)


def test_stand_ins_pass_gradcheck_in_fp64():
    rng = np.random.RandomState(3)
    a = torch.tensor([[-32.0, -32.0, 32.0, 32.0], [40.0, 8.0, 104.0, 72.0]], dtype=torch.float64)
    t = torch.tensor(rng.uniform(-1, 1, (2, 4)), dtype=torch.float64)
    d = torch.tensor(rng.uniform(-1, 1, (2, 4)), dtype=torch.float64, requires_grad=True)
    f = lambda d: 1 - O.giou_aligned(O.decode(a, d, STDS), O.decode(a, t, STDS))  # noqa: E731
    assert torch.autograd.gradcheck(f, (d,))
    z = torch.tensor(rng.standard_normal(5), dtype=torch.float64, requires_grad=True)
    tz = torch.tensor(rng.uniform(0, 1, 5), dtype=torch.float64)
    assert torch.autograd.gradcheck(
        lambda z: torch.nn.functional.binary_cross_entropy_with_logits(z, tz), (z,))
    x = torch.tensor(rng.standard_normal((4, 3)), dtype=torch.float64, requires_grad=True)
    lab = torch.tensor([0, 3, 2, 1])
    assert torch.autograd.gradcheck(lambda x: AO.sigmoid_focal_loss(x, lab), (x,))


def test_threshold_of_equal_ious_is_their_value():
    c = torch.full((45, 2), 0.3, dtype=torch.float32)
    c[:, 1] = 0.0
    assert O.threshold(c).tolist() == [np.float32(0.3), 0.0]


def test_constructor_keys_and_refusals():
    head = modules.LIGAATSSHead(**syn.KITTI_ATSS_HEAD)
    keys = set(head.state_dict())
    for k in ('cls_convs.0.conv.weight', 'cls_convs.3.gn.weight', 'cls_convs.3.gn.bias',
              'reg_convs.2.conv.weight', 'atss_cls.weight', 'atss_cls.bias', 'atss_reg.weight',
              'atss_centerness.bias', 'scales.4.scale'):
        assert k in keys, k
    assert 'cls_convs.0.conv.bias' not in keys
    assert head.atss_reg.out_channels == 12 and head.atss_cls.out_channels == 3
    cfg = modules._atss_loss_config(head)
    assert cfg['strides'] == [4, 8, 16, 32, 64] and cfg['loss_weight'] == [1.0, 2.0, 1.0]
    bad = [dict(reg_class_agnostic=True), dict(num_extra_reg_channel=2),
           dict(reg_avg_factor='sum_centerness'),
           dict(anchor_generator=dict(syn.KITTI_ATSS_HEAD['anchor_generator'], ratios=[0.5, 1.0])),
           dict(loss_bbox=dict(type='IoULoss', loss_weight=2.0)),
           dict(train_cfg=dict(syn.KITTI_ATSS_HEAD['train_cfg'],
                               assigner=dict(type='ATSS3DCenterAssigner', topk=9,
                                             thresh_mode='ratio'))),
           dict(train_cfg=dict(syn.KITTI_ATSS_HEAD['train_cfg'], append_3d_centers=False))]
    for kw in bad:
        with pytest.raises(NotImplementedError):
            modules._atss_loss_config(modules.LIGAATSSHead(**dict(syn.KITTI_ATSS_HEAD, **kw)))


# ---- GPU ----

TRAIN = (320, 1280)
FEAT = syn.atss_feat_sizes(*TRAIN)
WEIGHTS = (0.7, 1.3, 0.9)
KEYS = ('loss_cls', 'loss_bbox', 'loss_centerness')

# name -> (GT per image, pad shape per image)
CASES = {
    'b1_gt0': ([0], [TRAIN]),
    'b1_gt1': ([1], [TRAIN]),
    'b1_gt20': ([20], [TRAIN]),
    'b1_gt60': ([60], [TRAIN]),
    'b2_gt20_gt60': ([20, 60], [TRAIN, (288, 1216)]),
    'b2_gt0_gt1': ([0, 1], [(300, 1000), TRAIN]),
}


def _head():
    return modules.LIGAATSSHead(**syn.KITTI_ATSS_HEAD)


def _cuda_case(name, seed=31):
    ngt, pads = CASES[name]
    cls, box, ctr, gts, labels = syn.make_atss_loss_case(seed, FEAT, ngt, pads)
    outs = [[t.cuda().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
    return outs, [g.cuda() for g in gts], [lab.cuda() for lab in labels], pads


def _metas(pads):
    return [dict(pad_shape=(h, w, 3), img_shape=(h, w, 3)) for h, w in pads]


def _check_targets(helper, tg):
    """The targets of the last call against the fp32 restatement on the same device: assigned GT,
    labels, label weights and thresholds exactly, bbox and centerness targets within 2 ulp."""
    for k, dt in (('assigned_gt', torch.int32), ('labels', torch.int32),
                  ('label_weights', torch.float32)):
        want = torch.stack([t['assigned' if k == 'assigned_gt' else k] for t in tg]).to(dt)
        assert torch.equal(helper.debug_tensor(k), want), k
    thr = torch.cat([t['thresholds'] for t in tg])
    assert torch.equal(helper.debug_tensor('thresholds'), thr)
    for k in ('bbox_targets', 'centerness_targets'):
        got, want = helper.debug_tensor(k), torch.stack([t[k] for t in tg])
        ulp = torch.abs(torch.nextafter(want, torch.full_like(want, np.inf)) - want)
        assert bool((torch.abs(got - want) <= 2 * ulp).all()), k


def _weighted(losses, L):
    return sum(WEIGHTS[k] * (1 + lv / 10) * losses[key][lv]
               for k, key in enumerate(KEYS) for lv in range(L))


def _check(head, outs, gts, labels, pads, dtype=torch.float64, grad_rtol=1e-5):
    cfg = modules._atss_loss_config(head)
    flat = [t for ts in outs for t in ts]
    for t in flat:
        t.grad = None
    got = head.loss(*outs, gts, labels, _metas(pads))
    _weighted(got, len(FEAT)).backward()
    tg = O.targets(FEAT, cfg['strides'], cfg['octave_base_scale'], gts, labels, pads, cfg)
    _check_targets(head._atss_loss, tg)
    ins = [[t.detach().to(dtype).requires_grad_() for t in ts] for ts in outs]
    ref = O.losses(*ins, tg, FEAT, cfg['strides'], cfg['octave_base_scale'], cfg)
    for key in KEYS:
        for lv in range(len(FEAT)):
            assert got[key][lv].item() == pytest.approx(ref[key][lv].item(), rel=1e-6,
                                                        abs=1e-12), (key, lv)
    _weighted(ref, len(FEAT)).backward()
    for o, r in zip(flat, [t for ts in ins for t in ts]):
        torch.testing.assert_close(o.grad.to(dtype), r.grad, rtol=grad_rtol, atol=1e-7)
    return got, tg


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_loss_matches_the_restatement(name):
    outs, gts, labels, pads = _cuda_case(name)
    _check(_head(), outs, gts, labels, pads)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['b1_gt20', 'b2_gt20_gt60'])
def test_loss_on_the_heads_own_forward(name):
    _, gts, labels, pads = _cuda_case(name)
    torch.manual_seed(7)
    head = _head().cuda()
    B = len(pads)
    feats = [torch.randn(B, 64, h, w, device='cuda') for h, w in FEAT]
    cls, box, ctr = head(feats)
    for t in cls + box + ctr:
        t.retain_grad()
    _check(head, [cls, box, ctr], gts, labels, pads)
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all())
               for p in head.parameters())


def _small_case(gts, labels, pad=(64, 192), seed=5):
    feat = syn.atss_feat_sizes(*pad)
    cls, box, ctr, _, _ = syn.make_atss_loss_case(seed, feat, [0], [pad])
    outs = [[t.cuda().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
    return feat, outs, [torch.tensor(gts, dtype=torch.float32, device='cuda')], \
        [torch.tensor(labels, device='cuda')], [pad]


def _check_small(feat, outs, gts, labels, pads, dtype=torch.float64):
    global FEAT
    saved, FEAT = FEAT, feat
    try:
        return _check(_head(), outs, gts, labels, pads, dtype)
    finally:
        FEAT = saved


@pytest.mark.gpu
def test_distance_tie_at_the_ninth_candidate_keeps_the_lower_index():
    # the centre of a level-0 cell: 4 anchors at 2 sqrt(2), then 8 at sqrt(40); candidates 5-9
    # are 5 of those 8
    g = [[20.0, 10.0, 90.0, 50.0, 50.0, 26.0], [100.0, 4.0, 160.0, 60.0, 130.0, 34.0]]
    feat, outs, gts, labels, pads = _small_case(g, [0, 1])
    _, tg = _check_small(feat, outs, gts, labels, pads)
    assert all(t['num_pos'] > 0 for t in tg)


@pytest.mark.gpu
def test_gt_whose_candidate_ious_are_all_equal():
    # centre far to the left of the image: every candidate is in column 0, none reaches the box,
    # so all IoUs are 0, std 0, the threshold 0, and no candidate lies inside the box
    g = [[600.0, 100.0, 700.0, 200.0, -3000.0, 150.0], [200.0, 40.0, 400.0, 250.0, 300.0, 150.0]]
    cls, box, ctr, _, _ = syn.make_atss_loss_case(9, FEAT, [0], [TRAIN])
    outs = [[t.cuda().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
    gts = [torch.tensor(g, device='cuda')]
    labels = [torch.tensor([2, 1], device='cuda')]
    head = _head()
    _, tg = _check(head, outs, gts, labels, [TRAIN])
    assert head._atss_loss.debug_tensor('thresholds')[0].item() == 0.0
    assert not bool((tg[0]['assigned'] == 1).any()) and bool((tg[0]['assigned'] == 2).any())


@pytest.mark.gpu
def test_anchor_centre_at_the_in_gt_margin():
    # the anchors of column 0 have their centre at x = 0: a GT edge at -fp32(0.01) leaves them
    # exactly 0.01 inside (not positive), one ulp further out they are inside
    e = np.float32(0.01)
    res = []
    for x1 in (-e, -np.nextafter(e, np.float32(1))):
        g = [[float(x1), 20.0, 8.0, 60.0, 0.0, 40.0]]
        feat, outs, gts, labels, pads = _small_case(g, [1])
        _, tg = _check_small(feat, outs, gts, labels, pads)
        res.append(tg[0]['assigned'][10 * feat[0][1]].item())   # level 0, row 10, column 0
    assert res == [0, 1]


@pytest.mark.gpu
def test_predictions_on_the_size_clamp_and_at_their_targets():
    g = [[20.0, 10.0, 90.0, 50.0, 50.0, 30.0], [100.0, 4.0, 180.0, 60.0, 140.0, 30.0]]
    feat, outs, gts, labels, pads = _small_case(g, [0, 2])
    cfg = modules._atss_loss_config(_head())
    tg = O.targets(feat, cfg['strides'], cfg['octave_base_scale'], gts, labels, pads, cfg)
    r = np.float32(abs(math.log(16 / 1000)))
    # fp32 deltas whose size delta * 0.2 rounds onto the clamp, beyond it and inside it
    d = np.float32(r / np.float32(0.2))
    while np.float32(d * np.float32(0.2)) < r:
        d = np.nextafter(d, np.float32(np.inf))
    while np.float32(np.nextafter(d, np.float32(0)) * np.float32(0.2)) >= r:
        d = np.nextafter(d, np.float32(0))
    start = 0
    for lv, (h, w) in enumerate(feat):
        lab = tg[0]['labels'][start:start + h * w].view(h, w)
        t = tg[0]['bbox_targets'][start:start + h * w].view(h, w, 4)
        start += h * w
        with torch.no_grad():
            b = outs[1][lv].view(1, 4, 3, h, w)
            ys, xs = torch.nonzero(lab < 3, as_tuple=True)
            for i, (y, x) in enumerate(zip(ys.tolist(), xs.tolist())):
                c = lab[y, x].item()
                if i % 3 == 0:      # on the prediction's target: identical boxes
                    b[0, :, c, y, x] = t[y, x]
                elif i % 3 == 1:    # on the clamp, and beyond it
                    b[0, 2, c, y, x] = float(d)
                    b[0, 3, c, y, x] = -float(d) * 3
                else:               # far off: disjoint from the target
                    b[0, 0, c, y, x] = 80.0
    # the fp32 restatement: the fp64 one would move the clamp
    _check_small(feat, outs, gts, labels, pads, dtype=torch.float32)


@pytest.mark.gpu
def test_no_positive_anywhere_in_the_batch():
    g = [[600.0, 100.0, 700.0, 200.0, -3000.0, 150.0]]
    cls, box, ctr, _, _ = syn.make_atss_loss_case(9, FEAT, [0, 0], [TRAIN, TRAIN])
    outs = [[t.cuda().requires_grad_() for t in ts] for ts in (cls, box, ctr)]
    gts = [torch.tensor(g, device='cuda'), torch.zeros((0, 6), device='cuda')]
    labels = [torch.tensor([0], device='cuda'), torch.zeros(0, dtype=torch.long, device='cuda')]
    got, tg = _check(_head(), outs, gts, labels, [TRAIN, TRAIN])
    assert all(t['num_pos'] == 0 for t in tg)
    assert all(v.item() == 0.0 for v in got['loss_bbox'] + got['loss_centerness'])
    assert all(not bool(t.grad.any()) for t in outs[1] + outs[2])


@pytest.mark.gpu
def test_label_checks_and_gt_shape():
    outs, gts, labels, pads = _cuda_case('b2_gt20_gt60')
    head = _head()
    bad = [lab.clone() for lab in labels]
    bad[1][5] = 3
    with pytest.raises(ValueError):
        head.loss(*outs, gts, [b.cpu() for b in bad], _metas(pads))
    got = head.loss(*outs, gts, bad, _metas(pads))
    assert all(math.isnan(v.item()) for vs in got.values() for v in vs)
    got = head.loss(*outs, gts, labels, _metas(pads))
    assert all(math.isfinite(v.item()) for vs in got.values() for v in vs)
    with pytest.raises(RuntimeError):
        head.loss(*outs, [g[:, :4] for g in gts], labels, _metas(pads))
    with pytest.raises(NotImplementedError):
        head.loss(*outs, gts, labels, _metas(pads), gt_bboxes_ignore=[g[:1, :4] for g in gts])


@pytest.mark.gpu
def test_repeat_calls_are_bitwise_equal_without_host_synchronisation():
    outs, gts, labels, pads = _cuda_case('b2_gt20_gt60')
    head = _head()
    flat = [t for ts in outs for t in ts]
    head.loss(*outs, gts, labels, _metas(pads))      # creates the handle
    torch.cuda.synchronize()
    res = []
    for _ in range(2):
        for t in flat:
            t.grad = None
        torch.cuda.set_sync_debug_mode('error')
        try:
            got = head.loss(*outs, gts, labels, _metas(pads))
            _weighted(got, len(FEAT)).backward()
        finally:
            torch.cuda.set_sync_debug_mode('default')
        res.append([v.detach().clone() for vs in got.values() for v in vs] +
                   [t.grad.clone() for t in flat])
    for a, b in zip(*res):
        assert torch.equal(a, b)
    # without requires_grad no gradient buffer is written, and the losses do not change
    with torch.no_grad():
        got = head.loss(*[[t.detach() for t in ts] for ts in outs], gts, labels, _metas(pads))
    assert torch.equal(got['loss_cls'][0], res[0][0])
