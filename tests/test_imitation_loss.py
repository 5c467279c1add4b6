"""``DfMImitation.loss``: DfM's LiDAR imitation loss and its gradients.

CPU: the torch restatement (tests/imitation_loss_oracle.py) reproduces the reference's fixture
(tests/golden/imitation_loss.npz): mask and counts exactly, losses, gradients and scales within
fp32 bounds; the box test against hand-worked points; gradcheck; the layers, ``load_imitation``
and the refusals.  GPU: the native mask, counts, losses, gradients and scale update against the
fp64 restatement at the shipped KITTI shape, against the fixture, at the edges, and the call's
properties (bitwise repeats, no gradient unless asked, no host synchronisation)."""
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import checkpoint, modules
from depth_from_motion_b200 import synthetic as syn
from tests import imitation_loss_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'imitation_loss.npz')
KEYS = ('spatial_features_2d', 'volume_features')
IMITATION_CFGS = [
    dict(lidar_feature_layer='spatial_features_2d', stereo_feature_layer='spatial_features_2d',
         normalize='cw_scale', layer='conv2d', channel=64, kernel_size=1, use_relu=False,
         mode='inbox', loss_weight=1.0),
    dict(lidar_feature_layer='volume_features', stereo_feature_layer='volume_features',
         normalize='cw_scale', layer='conv3d', channel=32, kernel_size=1, use_relu=False,
         mode='inbox', loss_weight=1.0)]
GRAD_WEIGHTS = (1.0, 1.5)


def _shipped_cfg():
    import json
    m = json.load(open(os.path.join(HERE, 'golden', 'detector_configs.json')))[
        'dfm_r34_1x8_kitti-3d-3class.py']
    return m['imitation_cfgs'], m['bbox_head_3d']['anchor_generator'], \
        m['normalizer_clamp_value']


def _module(device='cpu'):
    cfgs, ag, clamp = _shipped_cfg()
    return modules.DfMImitation(cfgs, ag, clamp).to(device)


def golden_case(name):
    """The fixture case's inputs, regenerated: (case dict, inbox, initial scales, training)."""
    g = np.load(GOLDEN)
    seed, num_gt, kw, training = syn.IMITATION_GOLDEN_CASES[name]
    nz, ny, nx = syn.IMITATION_GOLDEN_SHAPE
    case = syn.make_imitation_case(seed, 1, num_gt, shape=(nz, ny, nx), **kw)
    _, ag, _ = _shipped_cfg()
    inbox = O.inbox_mask(*O.anchor_centres(ag, ny, nx), case['gt'])
    keep = syn.IMITATION_GOLDEN_KEEP.get(name)
    if keep is not None:
        for k, n in zip(KEYS, keep):
            O.keep_positives(case['teacher'][k], inbox, n)
    scales = [torch.from_numpy(g[f'{name}/init_scale_bev']),
              torch.from_numpy(g[f'{name}/init_scale_vol'])]
    return case, inbox, scales, training


def _oracle(case, inbox, scales, training, dtype, device='cpu'):
    """Restated losses, new scales, counts and (fp64) gradients of sum_i GRAD_WEIGHTS[i] loss_i."""
    xs = [case['stereo'][k].detach().to(device, dtype, copy=True).requires_grad_() for k in KEYS]
    ts = [case['teacher'][k].to(device) for k in KEYS]
    ps = [p.detach().to(device, dtype, copy=True).requires_grad_() for p in case['params']]
    losses, new, counts = O.imitation_loss(
        xs, ts, ps[0::2], ps[1::2], [s.to(device) for s in scales], inbox.to(device),
        [1.0, 1.0], 10.0, training)
    sum(w * l for w, l in zip(GRAD_WEIGHTS, losses)).backward()
    return losses, new, counts, [x.grad for x in xs], [p.grad for p in ps]


def _close(a, b, rel):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    scale = max(float(b.abs().max()) if b.numel() else 0.0, 1e-30)
    assert float((a - b).abs().max()) <= rel * scale, (float((a - b).abs().max()), scale)


# ---- CPU ----

@pytest.mark.parametrize('name', list(syn.IMITATION_GOLDEN_CASES))
def test_restatement_reproduces_reference_golden(name):
    g = np.load(GOLDEN)
    case, inbox, scales, training = golden_case(name)
    np.testing.assert_array_equal(inbox[0].numpy().astype(np.uint8), g[f'{name}/inbox'])
    l32, s32, counts, _, _ = _oracle(case, inbox, scales, training, torch.float32)
    assert counts == g[f'{name}/counts'].tolist()
    l64, _, _, gx, gp = _oracle(case, inbox, scales, training, torch.float64)
    l32, l64 = [v.detach() for v in l32], [v.detach() for v in l64]
    for i in range(2):
        assert float(l32[i]) == pytest.approx(float(g[f'{name}/loss_fp32'][i]), rel=1e-6, abs=0)
        assert float(l64[i]) == pytest.approx(float(g[f'{name}/loss_fp64'][i]), rel=1e-6, abs=0)
    for s, k in zip(s32, ('bev', 'vol')):
        want = torch.from_numpy(g[f'{name}/scale_{k}'])
        assert torch.equal(torch.isnan(s), torch.isnan(want))
        ok = ~torch.isnan(want)
        _close(s[ok], want[ok], 1e-6)
    for i, k in enumerate(('bev', 'vol')):
        _close(gx[i], g[f'{name}/grad_x_{k}'], 1e-6)
        _close(gp[2 * i].reshape(g[f'{name}/grad_w_{k}'].shape), g[f'{name}/grad_w_{k}'], 1e-6)
        _close(gp[2 * i + 1], g[f'{name}/grad_b_{k}'], 1e-6)


def test_fixture_pins_the_gate_clamp_and_nan_cases():
    g = np.load(GOLDEN)
    assert g['no_gt/counts'].tolist() == [0, 0] and not g['no_gt/loss_fp32'].any()
    assert g['gate_10_11/counts'].tolist() == [10, 11]
    # n = 10 leaves the BEV scale as it was, n = 11 updates the volume's
    assert np.array_equal(g['gate_10_11/scale_bev'], g['gate_10_11/init_scale_bev'])
    assert not np.array_equal(g['gate_10_11/scale_vol'], g['gate_10_11/init_scale_vol'])
    assert g['few_positives/counts'].tolist() == [4, 7]
    # the NaN teacher channels reach the scale in training mode only
    assert np.isnan(g['overlapping_rotated_nan/scale_bev']).any()
    assert np.array_equal(g['overlapping_rotated_nan_eval/scale_bev'],
                          g['overlapping_rotated_nan_eval/init_scale_bev'])
    assert np.isfinite(g['overlapping_rotated_nan/loss_fp32']).all()
    assert np.abs(g['overlapping_rotated_nan/gt'][:, 6]).max() > 0.1


def test_box_test_hand_worked_points():
    box = torch.tensor([[10.0, 5.0, -1.0, 4.0, 2.0, 1.5, 0.0]])
    edge = torch.tensor(12.0)                         # cx + dx / 2: on the edge, out
    inside = torch.nextafter(edge, torch.tensor(0.0))  # one fp32 ulp inside, in
    px = torch.stack([edge, inside, torch.tensor(10.0), torch.tensor(10.0),
                      torch.tensor(10.0)])
    py = torch.tensor([5.0, 5.0, 6.0, torch.nextafter(torch.tensor(6.0), torch.tensor(0.0)),
                       3.5])
    assert O.points_in_boxes_part(px, py, box).tolist() == [-1, 0, -1, 0, -1]
    # a quarter turn: dx lies along y
    rot = torch.tensor([[0.0, 0.0, 0.0, 4.0, 2.0, 1.0, float(np.float32(np.pi / 2))]])
    assert O.points_in_boxes_part(torch.tensor([0.0, 1.5, 0.0]), torch.tensor([1.9, 0.0, -0.5]),
                                  rot).tolist() == [0, -1, 0]
    # a negative height or a NaN box contains nothing; the first containing box wins
    two = torch.tensor([[0.0, 0.0, 0.0, 2.0, 2.0, -1.0, 0.0], [0.0, 0.0, 0.0, 2.0, 2.0, 1.0, 0.0],
                        [0.0, 0.0, 0.0, 4.0, 4.0, 1.0, 0.0]])
    assert O.points_in_boxes_part(torch.tensor([0.0, 1.5]), torch.tensor([0.0, 0.0]),
                                  two).tolist() == [1, 2]
    nan = torch.tensor([[float('nan'), 0.0, 0.0, 2.0, 2.0, 1.0, 0.0]])
    assert O.points_in_boxes_part(torch.tensor([0.0]), torch.tensor([0.0]), nan).tolist() == [-1]


def test_gradcheck_of_the_restatement():
    g = torch.Generator().manual_seed(3)
    B, ny, nx, nz = 2, 4, 5, 3
    xs = [torch.randn((B, 4, ny, nx), generator=g, dtype=torch.float64, requires_grad=True),
          torch.randn((B, 2, nz, ny, nx), generator=g, dtype=torch.float64, requires_grad=True)]
    ts = [torch.relu(torch.randn((B, 4, ny, nx), generator=g)),
          torch.relu(torch.randn((B, 2, nz, ny, nx), generator=g))]
    ws = [torch.randn((c, c), generator=g, dtype=torch.float64, requires_grad=True)
          for c in (4, 2)]
    bs = [torch.randn((c,), generator=g, dtype=torch.float64, requires_grad=True)
          for c in (4, 2)]
    scales = [torch.rand((1, c), generator=g) + 0.5 for c in (4, 2)]
    inbox = torch.rand((B, ny, nx), generator=g) < 0.6

    def f(x0, x1, w0, w1, b0, b1):
        losses, _, _ = O.imitation_loss([x0, x1], ts, [w0, w1], [b0, b1], scales, inbox,
                                        [1.0, 2.0], 10.0, False)
        return losses[0] + 0.5 * losses[1]

    assert torch.autograd.gradcheck(f, (*xs, *ws, *bs))


def test_layers_keep_the_reference_state_dict():
    m = _module()
    # _init_imitation_layers assigns norm_imitation before conv_imitation
    assert list(m.state_dict()) == [
        'norm_imitation.spatial_features_2d.scale', 'norm_imitation.volume_features.scale',
        'conv_imitation.0.weight', 'conv_imitation.0.bias', 'conv_imitation.1.weight',
        'conv_imitation.1.bias']
    assert tuple(m.conv_imitation[0].weight.shape) == (64, 64, 1, 1)
    assert tuple(m.conv_imitation[1].weight.shape) == (32, 32, 1, 1, 1)
    assert torch.equal(m.norm_imitation['volume_features'].scale, torch.ones(1, 32))
    single = modules.DfMImitation(IMITATION_CFGS[:1], syn.KITTI_ANCHOR_GENERATOR)
    assert list(single.state_dict())[1:] == ['conv_imitation.weight', 'conv_imitation.bias']


def _imitation_state(m, prefix='', seed=0):
    g = torch.Generator().manual_seed(seed)
    return OrderedDict((prefix + k, torch.randn(v.shape, generator=g))
                       for k, v in m.state_dict().items())


def test_load_imitation_from_mmdet3d_and_liga_checkpoints():
    m = _module()
    state = _imitation_state(m, seed=1)
    ckpt = dict(state_dict=OrderedDict(list(state.items()) + [
        ('backbone.conv1.weight', torch.zeros(1)), ('bbox_head_3d.conv_cls.bias', torch.zeros(1))]))
    res = checkpoint.load_imitation(ckpt, m)
    assert not res.missing_keys and not res.unexpected_keys
    for k, v in state.items():
        assert torch.equal(m.state_dict()[k], v)
    liga = OrderedDict((k.replace('conv_imitation', 'dense_head.conv_imitation')
                        .replace('norm_imitation', 'dense_head.norm_imitation'), v * 2)
                       for k, v in state.items())
    liga['global_step'] = torch.tensor(5)
    liga['dense_head.conv_cls.weight'] = torch.zeros(1)
    checkpoint.load_imitation(dict(model_state=liga), m)
    for k, v in state.items():
        assert torch.equal(m.state_dict()[k], v * 2)


def test_load_imitation_refuses_a_missing_key():
    m = _module()
    state = _imitation_state(m)
    del state['norm_imitation.volume_features.scale']
    with pytest.raises(RuntimeError, match='Missing key'):
        checkpoint.load_imitation(dict(state_dict=state), m)


@pytest.mark.parametrize('change', [
    dict(mode='full'), dict(kernel_size=3), dict(use_relu=True), dict(layer='none'),
    dict(normalize='scale'), dict(normalize=None), dict(channel=48)])
def test_unshipped_options_are_refused(change):
    cfgs = [dict(IMITATION_CFGS[0], **change), IMITATION_CFGS[1]]
    with pytest.raises(NotImplementedError):
        modules.DfMImitation(cfgs, syn.KITTI_ANCHOR_GENERATOR)


def test_cpu_tensors_are_refused():
    m = _module()
    case = syn.make_imitation_case(1, 1, 1, shape=(2, 8, 8))
    with pytest.raises(RuntimeError, match='CUDA'):
        m.loss(case['stereo'], case['teacher'], case['gt'])


def test_synthetic_case_is_sparse_with_gt_in_range():
    case = syn.make_imitation_case(5, 2, [3, 0], shape=(5, 64, 48), nan_rows=2)
    t = case['teacher']['volume_features']
    occupied = (t != 0).any(1).float().mean().item()
    assert 0.01 < occupied < 0.2
    assert int(torch.isnan(t).sum()) == 2
    assert [g.shape[0] for g in case['gt']] == [3, 0]
    gt = case['gt'][0]
    lo, hi = syn.KITTI_POINT_CLOUD_RANGE[:2], syn.KITTI_POINT_CLOUD_RANGE[3:5]
    assert ((gt[:, 0] >= lo[0]) & (gt[:, 0] <= hi[0]) & (gt[:, 1] >= lo[1]) &
            (gt[:, 1] <= hi[1])).all()


# ---- GPU ----

def _native(m, case, training=True, grads=True, device='cuda'):
    """Native losses, new scales and gradients (of sum_i GRAD_WEIGHTS[i] loss_i)."""
    m.train(training)
    xs = {k: case['stereo'][k].to(device).requires_grad_(grads) for k in KEYS}
    ts = {k: case['teacher'][k].to(device) for k in KEYS}
    with torch.no_grad():
        for conv, w, b in zip(m.conv_imitation, case['params'][0::2], case['params'][1::2]):
            conv.weight.copy_(w.view_as(conv.weight))
            conv.bias.copy_(b)
    for p in m.parameters():
        p.grad = None
        p.requires_grad_(grads)
    losses = m.loss(xs, ts, [g.to(device) for g in case['gt']])
    if grads:
        sum(w * l for w, l in zip(GRAD_WEIGHTS, losses)).backward()
    return losses, xs


def _check_against_oracle(m, case, scales, training=True):
    for k, s in zip(KEYS, scales):
        m.norm_imitation[k].scale.copy_(s)
    losses, xs = _native(m, case, training)
    _, ag, _ = _shipped_cfg()
    ny, nx = xs[KEYS[0]].shape[-2:]
    inbox = O.inbox_mask(*O.anchor_centres(ag, ny, nx, 'cuda'), [g.cuda() for g in case['gt']])
    assert torch.equal(m.debug_tensor('inbox').bool(), inbox)
    l64, new, counts, gx, gp = _oracle(case, inbox, scales, training, torch.float64, 'cuda')
    assert m.debug_tensor('counts').tolist() == counts
    for i in range(2):
        assert float(losses[i].detach()) == pytest.approx(float(l64[i].detach()), rel=1e-6,
                                                          abs=1e-30)
    for i, (k, conv) in enumerate(zip(KEYS, m.conv_imitation)):
        _close(xs[k].grad, gx[i], 1e-5)
        _close(conv.weight.grad.reshape(gp[2 * i].shape), gp[2 * i], 1e-5)
        _close(conv.bias.grad, gp[2 * i + 1], 1e-5)
        got = m.norm_imitation[k].scale
        if training:
            # a NaN teacher channel at a positive makes that channel's scale NaN, as in the
            # reference
            assert torch.equal(torch.isnan(got), torch.isnan(new[i]))
            ok = ~torch.isnan(new[i])
            _close(got[ok], new[i][ok], 1e-6)
        else:
            assert torch.equal(got, scales[i].cuda())
    return losses, counts


@pytest.mark.gpu
@pytest.mark.parametrize('batch,num_gt', [(1, 0), (1, 1), (1, 20), (1, 60), (2, 1), (2, 20),
                                          (2, 60), (2, (0, 20))])
def test_matches_fp64_restatement_at_shipped_shape(batch, num_gt):
    case = syn.make_imitation_case(700 + batch * 10 + (num_gt if isinstance(num_gt, int) else 7),
                                   batch, num_gt, nan_rows=3)
    g = torch.Generator().manual_seed(batch)
    scales = [torch.rand((1, c), generator=g) + 0.5 for c in (64, 32)]
    m = _module('cuda')
    _, counts = _check_against_oracle(m, case, scales, training=True)
    if num_gt not in (0, (0, 20)) or batch == 2:
        assert min(counts) > 0 or num_gt == 0


@pytest.mark.gpu
def test_eval_mode_leaves_the_scale_unchanged():
    case = syn.make_imitation_case(801, 2, 20)
    scales = [torch.full((1, 64), 0.7), torch.full((1, 32), 1.3)]
    _check_against_oracle(_module('cuda'), case, scales, training=False)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(syn.IMITATION_GOLDEN_CASES))
def test_matches_reference_golden(name):
    g = np.load(GOLDEN)
    case, inbox, scales, training = golden_case(name)
    m = _module('cuda')
    for k, s in zip(KEYS, scales):
        m.norm_imitation[k].scale.copy_(s)
    losses, xs = _native(m, case, training)
    assert torch.equal(m.debug_tensor('inbox').cpu(), torch.from_numpy(g[f'{name}/inbox'])[None])
    assert m.debug_tensor('counts').tolist() == g[f'{name}/counts'].tolist()
    for i in range(2):
        assert float(losses[i]) == pytest.approx(float(g[f'{name}/loss_fp64'][i]), rel=1e-6,
                                                 abs=1e-30)
    for i, (k, kk, conv) in enumerate(zip(KEYS, ('bev', 'vol'), m.conv_imitation)):
        _close(xs[k].grad, g[f'{name}/grad_x_{kk}'], 1e-5)
        _close(conv.weight.grad.reshape(g[f'{name}/grad_w_{kk}'].shape),
               g[f'{name}/grad_w_{kk}'], 1e-5)
        _close(conv.bias.grad, g[f'{name}/grad_b_{kk}'], 1e-5)
        want = torch.from_numpy(g[f'{name}/scale_{kk}'])
        got = m.norm_imitation[k].scale.cpu()
        assert torch.equal(torch.isnan(got), torch.isnan(want))
        _close(got[~torch.isnan(want)], want[~torch.isnan(want)], 1e-6)


def _axis_case(boxes, shape=(5, 304, 288), seed=11):
    case = syn.make_imitation_case(seed, 1, 0, shape=shape, occupancy=0.5)
    case['gt'] = [torch.tensor(boxes, dtype=torch.float32).reshape(-1, 7)]
    return case


@pytest.mark.gpu
def test_gt_edge_exactly_on_anchor_centres():
    ax, ay = O.anchor_centres(syn.KITTI_ANCHOR_GENERATOR, 304, 288)
    # a box whose x edges are anchor-centre columns 100 and 110 exactly (fp32): those columns are
    # out, 101..109 in; the y edges lie halfway between rows
    x0, x1 = float(ax[100]), float(ax[110])
    cx, dx = (x0 + x1) / 2, x1 - x0
    assert np.float32(cx) - np.float32(dx) / 2 == np.float32(x0)
    assert np.float32(cx) + np.float32(dx) / 2 == np.float32(x1)
    cy = float(ay[150] + ay[151]) / 2
    case = _axis_case([cx, cy, -1.0, dx, 1.0, 1.5, 0.0])
    m = _module('cuda')
    _native(m, case)
    inbox = m.debug_tensor('inbox')[0].bool().cpu()
    want = O.inbox_mask(ax, ay, case['gt'])[0]
    assert torch.equal(inbox, want)
    cols = torch.nonzero(inbox.any(0)).view(-1).tolist()
    assert cols == list(range(101, 110))


@pytest.mark.gpu
def test_zero_gt_gives_zero_loss_and_zero_gradients():
    m = _module('cuda')
    case = syn.make_imitation_case(12, 2, 0)
    losses, xs = _native(m, case)
    assert [float(v) for v in losses] == [0.0, 0.0]
    for k, conv in zip(KEYS, m.conv_imitation):
        assert not xs[k].grad.any() and not conv.weight.grad.any() and not conv.bias.grad.any()
    assert torch.equal(m.norm_imitation[KEYS[0]].scale, torch.ones(1, 64, device='cuda'))


@pytest.mark.gpu
def test_negative_height_and_nan_gt_contain_nothing():
    m = _module('cuda')
    box = [30.0, 0.0, -1.0, 6.0, 4.0, 1.5, 0.3]
    neg = [30.0, 0.0, -1.0, 6.0, 4.0, -1.5, 0.3]
    nan = [float('nan'), 0.0, -1.0, 6.0, 4.0, 1.5, 0.3]
    _native(m, _axis_case([box]))
    assert int(m.debug_tensor('inbox').sum()) > 0
    for b in (neg, nan):
        losses, _ = _native(m, _axis_case([b]))
        assert int(m.debug_tensor('inbox').sum()) == 0
        assert [float(v) for v in losses] == [0.0, 0.0]


@pytest.mark.gpu
def test_all_nan_teacher_channels():
    case = syn.make_imitation_case(13, 1, 20)
    t = case['teacher']['spatial_features_2d']
    t[:, 5] = torch.where(t[:, 5] != 0, torch.full_like(t[:, 5], float('nan')), t[:, 5])
    case['teacher']['volume_features'][:, 3] = float('nan')   # every row becomes positive
    m = _module('cuda')
    _, counts = _check_against_oracle(m, case, [torch.ones(1, 64), torch.ones(1, 32)])
    assert torch.isnan(m.norm_imitation[KEYS[1]].scale[0, 3])
    assert torch.isfinite(m.norm_imitation[KEYS[1]].scale[0, :3]).all()
    assert counts[1] == int(m.debug_tensor('inbox').sum()) * 5


@pytest.mark.gpu
@pytest.mark.parametrize('keep', [(10, 11), (11, 10), (3, 7), (0, 1)])
def test_update_gate_and_normaliser_clamp(keep):
    case = syn.make_imitation_case(14, 1, 20)
    _, ag, _ = _shipped_cfg()
    inbox = O.inbox_mask(*O.anchor_centres(ag, 304, 288), case['gt'])
    for k, n in zip(KEYS, keep):
        O.keep_positives(case['teacher'][k], inbox, n)
    scales = [torch.full((1, 64), 0.8), torch.full((1, 32), 1.2)]
    m = _module('cuda')
    losses, counts = _check_against_oracle(m, case, scales)
    assert counts == list(keep)
    for k, n, s in zip(KEYS, keep, scales):
        changed = not torch.equal(m.norm_imitation[k].scale.cpu(), s)
        assert changed == (n > 10)


@pytest.mark.gpu
def test_repeats_are_bitwise_equal_and_no_grad_buffers_without_requires_grad():
    case = syn.make_imitation_case(15, 2, 20)
    m = _module('cuda').eval()
    out = []
    for _ in range(2):
        losses, xs = _native(m, case, training=False)
        out.append([l.detach().clone() for l in losses] +
                   [xs[k].grad.clone() for k in KEYS] +
                   [p.grad.clone() for p in m.parameters()])
    for a, b in zip(*out):
        assert torch.equal(a, b)
    from depth_from_motion_b200 import capi
    capi.profile_enable(True)
    capi.profile_report()
    losses, xs = _native(m, case, training=False, grads=False)
    torch.cuda.synchronize()
    stages = capi.profile_report()
    capi.profile_enable(False)
    assert not any(l.requires_grad for l in losses)
    assert any(k.startswith('imitation_loss_forward') for k in stages)
    assert not any(k.startswith('imitation_loss_backward') for k in stages), stages
    assert [float(v) for v in losses] == [float(v) for v in out[0][:2]]


@pytest.mark.gpu
def test_only_the_weights_or_only_the_features():
    case = syn.make_imitation_case(16, 1, 20)
    m = _module('cuda')
    _, ref_x = _native(m, case)
    ref_w = [p.grad.clone() for p in m.parameters()]
    # features only
    xs = {k: case['stereo'][k].cuda().requires_grad_() for k in KEYS}
    for p in m.parameters():
        p.requires_grad_(False)
        p.grad = None
    m.norm_imitation[KEYS[0]].scale.fill_(1.0)
    m.norm_imitation[KEYS[1]].scale.fill_(1.0)
    m.train()
    losses = m.loss(xs, {k: case['teacher'][k].cuda() for k in KEYS},
                    [g.cuda() for g in case['gt']])
    sum(w * l for w, l in zip(GRAD_WEIGHTS, losses)).backward()
    for k in KEYS:
        assert torch.equal(xs[k].grad, ref_x[k].grad)
    assert all(p.grad is None for p in m.parameters())
    # weights only
    for p in m.parameters():
        p.requires_grad_(True)
    m.norm_imitation[KEYS[0]].scale.fill_(1.0)
    m.norm_imitation[KEYS[1]].scale.fill_(1.0)
    losses = m.loss({k: case['stereo'][k].cuda() for k in KEYS},
                    {k: case['teacher'][k].cuda() for k in KEYS}, [g.cuda() for g in case['gt']])
    sum(w * l for w, l in zip(GRAD_WEIGHTS, losses)).backward()
    for p, r in zip(m.parameters(), ref_w):
        assert torch.equal(p.grad, r)


@pytest.mark.gpu
def test_loss_and_backward_do_not_synchronise():
    case = syn.make_imitation_case(17, 2, 20)
    m = _module('cuda')
    _native(m, case)                                    # handle and anchors in place
    xs = {k: case['stereo'][k].cuda().requires_grad_() for k in KEYS}
    ts = {k: case['teacher'][k].cuda() for k in KEYS}
    gt = [g.cuda() for g in case['gt']]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        losses = m.loss(xs, ts, gt)
        (losses[0] + losses[1]).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert xs[KEYS[0]].grad is not None


@pytest.mark.gpu
def test_misshaped_and_mismatched_inputs_are_refused():
    case = syn.make_imitation_case(18, 2, 3, shape=(5, 32, 24))
    m = _module('cuda')
    xs = {k: case['stereo'][k].cuda() for k in KEYS}
    ts = {k: case['teacher'][k].cuda() for k in KEYS}
    gt = [g.cuda() for g in case['gt']]
    m.loss(xs, ts, gt)
    bad = [
        (dict(xs, volume_features=xs['volume_features'][:, :, :4]), ts, gt),
        (xs, dict(ts, spatial_features_2d=ts['spatial_features_2d'][:1]), gt),
        (dict(xs, spatial_features_2d=xs['spatial_features_2d'][:, :32]), ts, gt),
        (dict(xs, spatial_features_2d=xs['spatial_features_2d'].double()), ts, gt),
        (xs, dict(ts, volume_features=ts['volume_features'].cpu()), gt),
        (dict(xs, volume_features=xs['volume_features'][:1]),
         dict(ts, volume_features=ts['volume_features'][:1]), gt),
        ({KEYS[0]: xs[KEYS[0]]}, ts, gt),
        (xs, ts, gt[:1]),
        (xs, ts, [gt[0], gt[1][:, :6]]),
    ]
    for x, t, g in bad:
        with pytest.raises(RuntimeError):
            m.loss(x, t, g)


@pytest.mark.gpu
def test_workspace_is_small():
    m = _module('cuda')
    _native(m, syn.make_imitation_case(19, 2, 20))
    ws = m.workspace()
    feats = 2 * (64 + 32 * 5) * 304 * 288 * 4
    print(f'workspace {ws / 2**20:.2f} MiB against {feats / 2**20:.0f} MiB of stereo features')
    assert ws < 16 * 2**20


@pytest.mark.gpu
def test_on_native_frustum_and_hourglass_outputs():
    """The detector's own tensors: the native FrustumToVoxel volume and BEVHourglass BEV feature
    of a small synthetic case, built as DfM.forward_train builds them, are accepted."""
    import copy
    from oracle import dfm_oracle
    from tests import test_gpu_parity as P
    h, w, d = 64, 128, 16
    cur, prev, metas, params = syn.make_kitti_pair(23, h, w, d)
    cfg = syn.depth_cfg_for(d)
    fc = syn.make_frustum_case(24, h, w, d, (32, 28, 20))
    metas = copy.deepcopy(metas)
    metas[0]['cam2img'] = fc['metas'][0]['cam2img']
    bc = syn.make_bev_case(seed=25, nz=5, ny=28, nx=32)
    bb, fr = P._backbone(params, cfg, 'auto'), P._frustum_module(fc)
    bev, _ = P._bev_modules(bc)
    with torch.no_grad():
        cost, stereo, _ = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))
        lg = modules.CostLogits(cost, depth_samples=dfm_oracle.depth_samples(cfg))
        vol = fr(stereo, lg, metas, fc['sem'].cuda())
        _, nz, ny, nx = vol.shape[1:]
        _, feat = bev(vol.view(1, -1, ny, nx))
    assert vol.shape[1] == 32 and feat.shape[1] == 64
    case = syn.make_imitation_case(20, 1, 3, shape=(nz, ny, nx), size_scale=4.0, occupancy=0.5)
    case['stereo'] = dict(spatial_features_2d=feat.cpu(), volume_features=vol.cpu())
    _, counts = _check_against_oracle(_module('cuda'), case, [torch.ones(1, 64),
                                                              torch.ones(1, 32)])
    assert min(counts) > 0
