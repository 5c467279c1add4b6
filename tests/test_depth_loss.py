"""``DepthHead.loss``: DfM's dense depth loss and its gradient.

CPU: the torch restatement (tests/depth_loss_oracle.py) reproduces the reference's fixture
(tests/golden/depth_loss.npz) bit for bit in fp32; its column form agrees with the dense form in
fp64; the refusals.  GPU: the native loss, masked count and gradients against the fp64
restatement at the shipped training shape, against the fixture, and the call's properties
(bitwise repeats, no gradient unless asked, no host synchronisation, the empty case, workspace)."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import synthetic as syn
from oracle.ref_loader import reference_available
from tests import depth_loss_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'depth_loss.npz')


def _head(cfg, num_planes, f=4):
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=num_planes * f, min_depth=O.MIN_DEPTH,
                       max_depth=O.MAX_DEPTH), with_convs=False, depth_loss=cfg,
        downsample_factor=f, num_views=1)
    head.depth_samples = O.samples_for(num_planes, f)
    return head


def _upsample(cost, f=4):
    return F.interpolate(cost, scale_factor=f, mode='trilinear',
                         align_corners=True).flatten(start_dim=0, end_dim=1)


def _grad(t):
    return t.grad if t.grad is not None else torch.zeros_like(t)


# ---- CPU ----

@pytest.mark.parametrize('name', list(O.GOLDEN_CASES))
def test_restatement_reproduces_reference_golden(name):
    g = np.load(GOLDEN)
    cfg, cost, depth, fg, preds, samples = O.golden_inputs(name)
    leaf = cost.clone().requires_grad_()
    vol = _upsample(leaf)
    vol.retain_grad()
    loss = O.dense_loss(vol, depth, fg, samples, cfg, preds)
    assert loss.item() == g[f'{name}.loss'].item()
    if loss.requires_grad:
        loss.backward()
    np.testing.assert_array_equal(_grad(leaf).numpy(), g[f'{name}.grad_cost'])
    np.testing.assert_array_equal(_grad(vol).numpy(), g[f'{name}.grad_volume'])


@pytest.mark.skipif(not reference_available(), reason='needs the reference tree')
def test_regenerated_fixture_is_bitwise_equal():
    spec = importlib.util.spec_from_file_location(
        'make_depth_loss_golden', os.path.join(HERE, 'golden', 'make_depth_loss_golden.py'))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(GOLDEN)
    for name in O.GOLDEN_CASES:
        for k, v in mk.run_reference(name).items():
            np.testing.assert_array_equal(v, g[f'{name}.{k}'], err_msg=f'{name}.{k}')


def test_fixture_pins_the_edge_cases():
    cfg, cost, depth, fg, preds, samples = O.golden_inputs('edges_focal')
    mask = (depth > O.MIN_DEPTH) & (depth < O.MAX_DEPTH)
    assert not mask[0].any() and mask[1].any()
    e = torch.from_numpy(O.edge_depths(samples))
    got = mask[1, 3, 5:5 + len(e)].tolist()
    # fp32(min) and fp32(max) are outside, their inward nextafter inside, outward outside
    assert got[:6] == [False, True, False, False, True, False]
    assert all(got[6:])
    assert float(np.float32(O.MAX_DEPTH)) != O.MAX_DEPTH   # the bound compares as fp32
    # a gt on a bin centre: the neighbours' weight follows the fp32 formula
    interval = samples[1] - samples[0]
    p = 1 - (torch.abs(samples - samples[7]) / interval).clamp(max=1.0)
    assert p[7].item() == 1.0 and (p > 0).sum().item() <= 3


@pytest.mark.parametrize('name', [n for n in O.GOLDEN_CASES if n != 'no_masked_pixel'])
def test_column_form_matches_dense_form_in_fp64(name):
    cfg, cost, depth, fg, preds, samples = O.golden_inputs(name)
    a = cost.double().requires_grad_()
    b = cost.double().requires_grad_()
    dense = O.dense_loss(_upsample(a), depth, fg, samples, cfg, preds.double())
    col = O.column_loss(b, depth, fg, samples, cfg, preds.double())
    dense.backward()
    col.backward()
    assert col.item() == pytest.approx(dense.item(), rel=1e-12)
    tol = 1e-12 * a.grad.abs().max().item()
    assert (a.grad - b.grad).abs().max().item() <= tol


@pytest.mark.parametrize('kind', ['l1', 'purel1', 'gaussian_1.0', 'laplacian_1.0', 'hard_ce'])
def test_other_loss_types_are_refused(kind):
    head = _head(dict(type=kind, loss_weight=1.0), 8)
    cfg, cost, depth, fg, preds, _ = O.golden_inputs('ce')
    with pytest.raises(NotImplementedError, match='balanced_focal'):
        head.loss(preds, modules.CostLogits(cost), depth, fg)


@pytest.mark.parametrize('kind', ['balanced_ce', 'balanced_focal'])
def test_balanced_types_need_the_foreground_mask(kind):
    head = _head(O.loss_config(kind), 8)
    cfg, cost, depth, fg, preds, _ = O.golden_inputs('ce')
    with pytest.raises(ValueError):
        head.loss(preds, modules.CostLogits(cost), depth)


def test_misshaped_inputs_are_refused():
    head = _head(O.SHIPPED_LOSS, 8)
    cfg, cost, depth, fg, preds, _ = O.golden_inputs('ce')
    with pytest.raises(RuntimeError, match='depth_img'):
        head.loss(preds, modules.CostLogits(cost), depth[:, :-1], fg)
    with pytest.raises(RuntimeError, match='depth_fgmask_img'):
        head.loss(preds, modules.CostLogits(cost), depth, fg[:1])
    with pytest.raises(RuntimeError, match='depth_preds'):
        head.loss(preds[:, :, :-4], modules.CostLogits(cost), depth, fg)
    with pytest.raises(RuntimeError, match='depth_samples'):      # 7 planes for 8 * 4 samples
        head.loss(preds, modules.CostLogits(cost[:, :, :7]), depth, fg)
    with pytest.raises(RuntimeError, match='depth_samples'):      # dense: 30 bins
        head.loss(preds, _upsample(cost)[:, :30], depth, fg)


def test_synthetic_case_is_sparse_and_reaches_outside_the_range():
    cost, depth, fg = syn.make_depth_loss_case(0, 1, 72, 80, 320, 4, 0.05)
    assert cost.shape == (1, 1, 72, 80, 320) and fg.dtype == torch.int32
    assert 10 < cost.abs().max().item() < 40
    valid = depth > 0
    assert 0.03 < valid.float().mean().item() < 0.07
    d = depth[valid]
    assert (d < O.MIN_DEPTH).any() and (d > O.MAX_DEPTH).any()


# ---- GPU ----

SHIPPED = dict(D=72, H=80, W=320, f=4)     # KITTI training crop 320 x 1280


def _shipped_case(n, density=0.05, seed=21):
    cost, depth, fg = syn.make_depth_loss_case(seed, n, SHIPPED['D'], SHIPPED['H'],
                                               SHIPPED['W'], SHIPPED['f'], density)
    preds = torch.full(depth.shape, 30.0)
    return [t.cuda() for t in (cost, depth, fg, preds)]


def _native(head, form, cost, depth, fg, preds):
    """(loss, gradient with respect to the form's input, that input)."""
    if form == 'logits':
        x = cost.clone().requires_grad_()
        loss = head.loss(preds, modules.CostLogits(x), depth, fg)
    else:
        x = _upsample(cost).detach().requires_grad_()
        loss = head.loss(preds, x, depth, fg)
    loss.backward()
    return loss.detach(), x.grad, x


def _restated(cfg, form, x, depth, fg, preds, samples, dtype):
    """The restatement in ``dtype``; the logits form with fp32 interpolation weights, those of
    the fp32 volume the reference builds (see ``column_loss``)."""
    x = x.detach().to(dtype).requires_grad_()
    if form == 'logits':
        loss = O.column_loss(x, depth, fg, samples, cfg, preds.to(dtype),
                             weights_dtype=torch.float32)
    else:
        loss = O.dense_loss(x, depth, fg, samples, cfg, preds.to(dtype))
    loss.backward()
    return loss.detach(), x.grad


GPU_CASES = [(n, t, form, 0.05) for n in (1, 2) for t in O.TYPES for form in ('logits', 'dense')]
GPU_CASES.append((1, 'balanced_focal', 'logits', 1.0))


@pytest.mark.gpu
@pytest.mark.parametrize('n,kind,form,density', GPU_CASES)
def test_matches_fp64_restatement_at_shipped_shape(n, kind, form, density):
    cfg = O.loss_config(kind)
    head = _head(cfg, SHIPPED['D'])
    cost, depth, fg, preds = _shipped_case(n, density)
    samples = head.depth_samples.cuda()
    loss, grad, x = _native(head, form, cost, depth, fg, preds)
    mask = (depth > O.MIN_DEPTH) & (depth < O.MAX_DEPTH)
    assert head._depth_loss.debug_tensor('count').item() == int(mask.sum())
    l64, g64 = _restated(cfg, form, x, depth, fg, preds, samples, torch.float64)
    # the fp32 restatement: the reference's own arithmetic (dense upsampling for the logits)
    if form == 'logits':
        xr = x.detach().clone().requires_grad_()
        l32 = O.dense_loss(_upsample(xr), depth, fg, samples, cfg, preds)
        l32.backward()
        l32, g32 = l32.detach(), xr.grad
    else:
        l32, g32 = _restated(cfg, form, x, depth, fg, preds, samples, torch.float32)
    gmax = g64.abs().max().item()
    dev_loss = abs(loss.item() - l64.item()) / abs(l64.item())
    dev_grad = (grad.double() - g64).abs().max().item() / gmax
    print(f'{n} {kind} {form} density {density}: native loss rel {dev_loss:.2e}, grad '
          f'{dev_grad:.2e} of max; fp32 restatement loss rel '
          f'{abs(l32.item() - l64.item()) / abs(l64.item()):.2e}, grad '
          f'{(g32.double() - g64).abs().max().item() / gmax:.2e} of max (bounds 1e-5)')
    assert dev_loss <= 1e-5
    assert dev_grad <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['logits', 'dense'])
@pytest.mark.parametrize('name', list(O.GOLDEN_CASES))
def test_matches_reference_golden(name, form):
    g = np.load(GOLDEN)
    cfg, cost, depth, fg, preds, samples = O.golden_inputs(name)
    head = _head(cfg, O.GOLDEN_SHAPE['D'])
    loss, grad, _ = _native(head, form, *(t.cuda() for t in (cost, depth, fg, preds)))
    want = g[f'{name}.loss'].item()
    assert loss.item() == pytest.approx(want, rel=1e-6, abs=1e-30)
    ref = g[f'{name}.grad_cost' if form == 'logits' else f'{name}.grad_volume']
    tol = 1e-6 * np.abs(ref).max()
    np.testing.assert_array_less(np.abs(grad.cpu().numpy() - ref), tol + 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['logits', 'dense'])
def test_repeated_calls_are_bitwise_equal(form):
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    case = _shipped_case(2)
    l1, g1, _ = _native(head, form, *case)
    l2, g2, _ = _native(head, form, *case)
    assert torch.equal(l1, l2) and torch.equal(g1, g2)


@pytest.mark.gpu
def test_no_gradient_pass_without_requires_grad():
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    cost, depth, fg, preds = _shipped_case(1)
    with_grad, _, _ = _native(head, 'logits', cost, depth, fg, preds)
    capi.profile_enable(True)
    capi.profile_report()
    try:
        loss = head.loss(preds, modules.CostLogits(cost), depth, fg)
        torch.cuda.synchronize()
        stages = capi.profile_report()
    finally:
        capi.profile_enable(False)
    assert not loss.requires_grad
    assert torch.equal(loss, with_grad)
    assert any(k.startswith('depth_loss_pixel') for k in stages)
    assert not any(k.startswith('depth_loss_adjoint') for k in stages), stages


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['logits', 'dense'])
def test_loss_and_backward_do_not_synchronise(form):
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    case = _shipped_case(1)
    _native(head, form, *case)                    # handle and device samples in place
    x = case[0].clone().requires_grad_() if form == 'logits' else \
        _upsample(case[0]).detach().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        vol = modules.CostLogits(x) if form == 'logits' else x
        head.loss(case[3], vol, case[1], case[2]).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert x.grad is not None


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['logits', 'dense'])
def test_no_masked_pixel(form):
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    cost, depth, fg, preds = _shipped_case(2)
    depth = torch.where(depth < 1.0, depth, torch.full_like(depth, 70.0))
    loss, grad, _ = _native(head, form, cost, depth, fg, preds)
    assert loss.item() == 0.0 and not grad.any()
    assert head._depth_loss.debug_tensor('count').item() == 0
    preds[1, 5, 7] = float('nan')
    loss, grad, _ = _native(head, form, cost, depth, fg, preds)
    assert torch.isnan(loss) and not grad.any()


@pytest.mark.gpu
def test_workspace_is_far_below_the_dense_volume():
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    _native(head, 'logits', *_shipped_case(1))
    dense = 288 * 320 * 1280 * 4
    ws = head._depth_loss.workspace()
    print(f'workspace {ws / 2**20:.1f} MiB against the {dense / 2**20:.0f} MiB dense volume')
    assert ws < dense / 16


@pytest.mark.gpu
def test_per_pixel_loss_sums_to_the_loss():
    head = _head(O.SHIPPED_LOSS, SHIPPED['D'])
    cost, depth, fg, preds = _shipped_case(2)
    loss, _, _ = _native(head, 'logits', cost, depth, fg, preds)
    pix = head._depth_loss.debug_tensor('pixel_loss').view(depth.shape)
    mask = (depth > O.MIN_DEPTH) & (depth < O.MAX_DEPTH)
    assert not pix[~mask].any()
    assert pix.double().sum().item() / int(mask.sum()) == pytest.approx(loss.item(), rel=1e-6)


@pytest.mark.gpu
def test_on_native_backbone_cost():
    from oracle import dfm_oracle
    d = 24
    cur, prev, metas, params = syn.make_kitti_pair(3, 64, 192, d)
    dcfg = syn.depth_cfg_for(d)
    bb = modules.DfMBackbone(in_channels=32, depth_cfg=dcfg).to('cuda').eval()
    bb.load_state_dict(params, strict=True)
    bb.downsampled_depth = dfm_oracle.downsampled_depth(dcfg)
    with torch.no_grad():
        cost = bb(cur.cuda(), prev.cuda(), copy.deepcopy(metas))[0]
    assert cost.shape[:3] == (1, 1, d)
    h, w = cost.shape[3:]
    _, depth, fg = syn.make_depth_loss_case(4, 1, d, h, w, 4, 0.3)
    depth, fg = depth.cuda(), fg.cuda()
    preds = torch.zeros_like(depth)
    head = _head(O.SHIPPED_LOSS, d)
    loss, grad, x = _native(head, 'logits', cost, depth, fg, preds)
    l64, g64 = _restated(O.SHIPPED_LOSS, 'logits', x, depth, fg, preds,
                         head.depth_samples.cuda(), torch.float64)
    assert loss.item() == pytest.approx(l64.item(), rel=1e-5)
    assert (grad.double() - g64).abs().max().item() <= 1e-5 * g64.abs().max().item()
