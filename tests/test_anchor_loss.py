"""Training loss of both anchor heads (``LIGAAnchor3DHead.loss`` / ``Anchor3DHead.loss``).

CPU: the restatement's mmcv / mmdet stand-ins against hand-worked values and central finite
differences, LIGA's all-reduced ``avg_factor`` over two gloo ranks.  GPU: the native targets,
loss values and gradients against the restatement (tests/anchor_loss_oracle.py) at the shipped
grids and configs."""
import math

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import modules
from depth_from_motion_b200 import synthetic as syn
from tests import anchor_loss_oracle as O


# ---- CPU: the stand-ins ----

def test_focal_matches_hand_values_in_the_flt_min_clamp():
    # x = -200: p rounds to 0 in fp32, so the target log reads log(FLT_MIN)
    x = torch.tensor([[-200.0, 0.0]], requires_grad=True)
    t = torch.tensor([0])
    loss = O.sigmoid_focal_loss(x, t)
    lmin = math.log(O.FLT_MIN)
    assert loss[0, 0].item() == pytest.approx(-0.25 * lmin, rel=1e-6)
    # x = 0, not the target: -(1 - a) p^g log(1 - p) with p = 1/2
    assert loss[0, 1].item() == pytest.approx(-0.75 * 0.25 * math.log(0.5), rel=1e-6)
    loss.sum().backward()
    # target, p = 0: -a (1 - p)^g (1 - p - g p log p) = -a
    assert x.grad[0, 0].item() == pytest.approx(-0.25, rel=1e-6)
    # not the target, p = 1/2: -(1 - a) p^g (g (1 - p) log(1 - p) - p)
    assert x.grad[0, 1].item() == pytest.approx(-0.75 * 0.25 * (2 * 0.5 * math.log(0.5) - 0.5),
                                                rel=1e-6)


def test_iou3d_of_boxes_a_right_angle_apart_and_sharing_an_edge():
    a = torch.tensor([[0., 0., 0., 4., 2., 1., 0.]], dtype=torch.float64)
    b = torch.tensor([[0., 0., 0., 4., 2., 1., np.pi / 2]], dtype=torch.float64)
    # BEV overlap 2 x 2, volumes 8: 4 / (8 + 8 - 4) (mmcv's 1e-8 in the crossing parameter
    # moves it by ~1e-9)
    assert O.diff_iou_rotated_3d(a, b).item() == pytest.approx(1 / 3, rel=1e-7)
    c = torch.tensor([[4., 0., 0., 4., 2., 1., 0.]], dtype=torch.float64)
    assert O.diff_iou_rotated_3d(a, c).item() == pytest.approx(0.0, abs=1e-12)
    d = torch.tensor([[0., 0., 0.5, 4., 2., 1., 0.]], dtype=torch.float64)
    assert O.diff_iou_rotated_3d(a, d).item() == pytest.approx(4 / 12, rel=1e-9)


def test_iou3d_gradient_matches_central_differences():
    rng = np.random.RandomState(5)
    p = np.array([[0.3, -0.2, 0.1, 3.9, 1.7, 1.5, 0.35], [1.0, 2.0, -0.3, 0.9, 0.7, 1.8, -1.2],
                  [0.0, 0.0, 0.0, 2.0, 1.0, 1.0, 0.8]])
    t = p + rng.uniform(-0.3, 0.3, p.shape)
    t[:, 3:6] = np.abs(t[:, 3:6])
    pt = torch.tensor(p, requires_grad=True)
    tt = torch.tensor(t)
    O.diff_iou_rotated_3d(pt, tt).sum().backward()
    h = 1e-6
    for i in range(p.shape[0]):
        for k in range(7):
            e = np.zeros_like(p)
            e[i, k] = h
            f = lambda q: O.diff_iou_rotated_3d(torch.tensor(q), tt)[i].item()  # noqa: E731
            fd = (f(p + e) - f(p - e)) / (2 * h)
            assert pt.grad[i, k].item() == pytest.approx(fd, rel=1e-5, abs=1e-8), (i, k)


def test_assigner_tie_and_low_quality_rules():
    # GT 0 and 1 tie at anchor 0: the argmax takes GT 0, the low-quality pass then gives the
    # anchor to GT 1 (later GT win); anchor 1 (max 0.4, ignored) becomes GT 2's low-quality
    # match; anchor 2 stays negative
    ov = torch.tensor([[0.7, 0.2, 0.30], [0.7, 0.1, 0.05], [0.0, 0.40, 0.1]])
    asg = O.max_iou_assign(ov, 0.6, 0.35, 0.35)
    assert asg.tolist() == [2, 3, 0]
    # a GT whose best IoU is below min_pos_iou gets no low-quality match
    asg = O.max_iou_assign(torch.tensor([[0.3, 0.2]]), 0.6, 0.35, 0.35)
    assert asg.tolist() == [0, 0]


def _dist_worker(rank, port, out):
    import torch.distributed as dist
    dist.init_process_group('gloo', init_method=f'tcp://127.0.0.1:{port}', rank=rank,
                            world_size=2)
    v = modules._dist_reduce_mean(torch.tensor([3.0 + 4.0 * rank]))
    out[rank] = v.item()
    dist.destroy_process_group()


def test_liga_avg_factor_is_the_all_reduced_mean_over_two_ranks():
    import torch.multiprocessing as mp
    import socket
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_dist_worker, args=(port, out), nprocs=2, join=True)
    assert out[0] == out[1] == 5.0
    # one process without torch.distributed: the count itself
    assert modules._dist_reduce_mean(torch.tensor([7.0])).item() == 7.0


def test_unsupported_options_raise():
    head = _waymo_head()
    head.extra_cfg['loss_cls'] = dict(type='CrossEntropyLoss', use_sigmoid=True)
    with pytest.raises(NotImplementedError):
        modules._loss_config(head, False)
    head = _waymo_head()
    head.train_cfg = dict(syn.WAYMO_TRAIN_CFG, code_weight=[1.0] * 7)
    with pytest.raises(NotImplementedError):
        modules._loss_config(head, False)
    head = _kitti_head()
    head.train_cfg = dict(syn.KITTI_TRAIN_CFG, assigner=syn.KITTI_TRAIN_CFG['assigner'][:2])
    with pytest.raises(NotImplementedError):
        modules._loss_config(head, True)
    cfg = modules._loss_config(_kitti_head(), True)
    assert cfg['assign_per_class'] and cfg['with_iou'] and cfg['reduce_avg_factor']
    assert cfg['loss_weight'] == [1.0, 0.5, 0.2, 1.0]


# ---- GPU ----

def _kitti_head():
    return modules.LIGAAnchor3DHead(
        num_classes=3, in_channels=64, feat_channels=64, norm_cfg=dict(type='GN', num_groups=32),
        anchor_generator=syn.KITTI_ANCHOR_GENERATOR, dir_offset=syn.KITTI_DIR_OFFSET,
        assign_per_class=True, diff_rad_by_sin=True, train_cfg=syn.KITTI_TRAIN_CFG,
        test_cfg=syn.KITTI_TEST_CFG, **syn.KITTI_LOSSES)


def _waymo_head():
    return modules.Anchor3DHead(
        num_classes=3, in_channels=256, anchor_generator=syn.WAYMO_ANCHOR_GENERATOR,
        dir_offset=syn.WAYMO_DIR_OFFSET, train_cfg=syn.WAYMO_TRAIN_CFG,
        test_cfg=syn.WAYMO_TEST_CFG, **syn.WAYMO_LOSSES)


# name -> (head, liga, ny, nx, GT per sample, case arguments)
CASES = {
    'kitti_b1': (_kitti_head, True, 304, 288, [20], {}),
    'kitti_b1_class_without_gt': (_kitti_head, True, 304, 288, [16], dict(drop_class=2)),
    'kitti_b2_one_empty': (_kitti_head, True, 304, 288, [18, 0], {}),
    'kitti_zero_positives': (_kitti_head, True, 304, 288, [0], {}),
    'waymo_b1': (_waymo_head, False, 300, 220, [250], dict(cross_class=True)),
    'waymo_b2': (_waymo_head, False, 300, 220, [250, 240], dict(cross_class=True)),
    'waymo_b2_one_empty': (_waymo_head, False, 300, 220, [0, 60], {}),
}


def _run_case(name, seed=11):
    make, liga, ny, nx, ngt, kw = CASES[name]
    head = make()
    cfg = modules._loss_config(head, liga)
    dev = torch.device('cuda')
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, dev)
    cls, box, dirc, gts, labels = syn.make_anchor_loss_case(
        seed, anchors.cpu().numpy(), ny, nx, cfg['num_sizes'], cfg['num_rots'],
        cfg['num_classes'], ngt, **kw)
    cls, box, dirc = (t.to(dev).requires_grad_() for t in (cls, box, dirc))
    gts = [g.to(dev) for g in gts]
    labels = [lab.to(dev) for lab in labels]
    metas = [{} for _ in ngt]
    return head, liga, cfg, anchors, (cls, box, dirc), gts, labels, metas


def _oracle(cfg, anchors, outs, gts, labels, dtype):
    tg = O.targets(anchors, cfg['num_sizes'], cfg['num_rots'], gts, labels, cfg)
    ins = [t.detach().to(dtype).requires_grad_() for t in outs]
    return tg, ins, O.losses(*ins, tg, anchors, cfg)


WEIGHTS = (0.7, 1.3, 0.9, 1.1)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_loss_matches_the_restatement(name):
    _check_against_restatement(name, *_run_case(name))


def _check_against_restatement(name, head, liga, cfg, anchors, outs, gts, labels, metas):
    got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, labels, metas)
    keys = ['loss_cls', 'loss_bbox', 'loss_dir'] + (['loss_iou'] if cfg['with_iou'] else [])
    assert sorted(got) == sorted(keys)
    total = sum(w * got[k][0] for w, k in zip(WEIGHTS, keys))
    total.backward()
    helper = head._anchor_loss
    tg, ins, ref = _oracle(cfg, anchors, outs, gts, labels, torch.float64)
    # targets: the fp32 restatement on the same device, exactly (bbox targets within 2 ulp)
    for k, dt in (('assigned_gt', torch.int32), ('labels', torch.int32),
                  ('label_weights', torch.float32), ('dir_targets', torch.int32)):
        want = torch.stack([t['assigned' if k == 'assigned_gt' else k] for t in tg]).to(dt)
        assert torch.equal(helper.debug_tensor(k), want), k
    bt = helper.debug_tensor('bbox_targets')
    want = torch.stack([t['bbox_targets'] for t in tg])
    ulp = torch.abs(torch.nextafter(want, torch.full_like(want, np.inf)) - want)
    assert bool((torch.abs(bt - want) <= 2 * ulp).all())
    # loss values against fp64
    for k in keys:
        assert got[k][0].item() == pytest.approx(ref[k].item(), rel=1e-6, abs=1e-12), k
    # gradients against fp64 autograd with mmcv's focal backward
    rtotal = sum(w * ref[k] for w, k in zip(WEIGHTS, keys))
    rtotal.backward()
    for o, r, nm in zip(outs, ins, ('cls', 'bbox', 'dir')):
        torch.testing.assert_close(o.grad.double(), r.grad, rtol=1e-5, atol=1e-7,
                                   msg=lambda m: f'{name} grad {nm}: {m}')


@pytest.mark.gpu
def test_two_calls_are_bitwise_equal_and_no_grad_runs():
    head, liga, cfg, anchors, outs, gts, labels, metas = _run_case('waymo_b2')
    res = []
    for _ in range(2):
        for o in outs:
            o.grad = None
        got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, labels, metas)
        sum(v[0] for v in got.values()).backward()
        res.append([v[0].detach().clone() for v in got.values()] + [o.grad.clone() for o in outs])
    for a, b in zip(*res):
        assert torch.equal(a, b)
    with torch.no_grad():
        got = head.loss([o.detach() for o in outs[:1]], [outs[1].detach()], [outs[2].detach()],
                        gts, labels, metas)
    assert torch.equal(got['loss_cls'][0], res[0][0])


@pytest.mark.gpu
def test_iou_loss_stays_finite_at_degenerate_geometry():
    head, liga, cfg, anchors, outs, gts, labels, metas = _run_case('kitti_b1')
    # GT exactly on anchors, predictions of zero deltas: identical boxes; then nested, disjoint,
    # edge-touching and zero height overlap through the predicted deltas
    an = anchors.view(304, 288, 6, 7)
    g = torch.stack([an[100, 100, 0], an[120, 140, 1], an[200, 40, 2]])
    lab = torch.tensor([0, 1, 2], device='cuda')
    cls, box, dirc = (o.detach().clone() for o in outs)
    for fill in ([0.0] * 7, [0.0, 0.0, 0.0, -0.5, -0.5, 0.0, 0.0], [3.0, 0, 0, 0, 0, 0, 0],
                 [0.0, 0.0, 5.0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0, 1.5707964]):
        box.view(1, 6, 7, 304, 288)[:] = torch.tensor(fill, device='cuda')[None, None, :, None,
                                                                             None]
        b = box.clone().requires_grad_()
        got = head.loss([cls], [b], [dirc], [g], [lab], metas)
        got['loss_iou'][0].backward()
        assert math.isfinite(got['loss_iou'][0].item()), fill
        assert bool(torch.isfinite(b.grad).all()), fill


@pytest.mark.gpu
def test_out_of_range_labels_are_refused_or_poison_the_loss():
    head, liga, cfg, anchors, outs, gts, labels, metas = _run_case('waymo_b2_one_empty')
    bad = [lab.clone() for lab in labels]
    bad[1][3] = 3
    with pytest.raises(ValueError):
        head.loss([outs[0]], [outs[1]], [outs[2]], gts, [b.cpu() for b in bad], metas)
    got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, bad, metas)
    assert all(math.isnan(v[0].item()) for v in got.values())
    got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, labels, metas)
    assert all(math.isfinite(v[0].item()) for v in got.values())


def _native_head_outputs(head, c, ny, nx, seed):
    """The head's own CUDA forward, random conv weights (fan-in scaled), a random BEV map."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in head.named_parameters():
            if n.endswith('weight') and p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p[0].numel()))
    head = head.cuda().eval()
    x = torch.randn((1, c, ny, nx), generator=g).cuda()
    with torch.no_grad():
        cls, box, dirc = (t[0] for t in head([x]))
    return head, [t.requires_grad_() for t in (cls, box, dirc)]


@pytest.mark.gpu
@pytest.mark.parametrize('name,c', [('kitti_b1', 64), ('waymo_b1', 256)])
def test_loss_on_native_head_outputs(name, c):
    head, liga, cfg, anchors, outs, gts, labels, metas = _run_case(name)
    ny, nx = outs[0].shape[-2:]
    head, outs = _native_head_outputs(head, c, ny, nx, seed=23)
    _check_against_restatement(name + '_native', head, liga, cfg, anchors, outs, gts, labels,
                               metas)
