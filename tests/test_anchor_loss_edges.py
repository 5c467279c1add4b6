"""Training loss of both anchor heads at its fp32 decision edges.

The cases put the kernel's discrete decisions on, or within a few ulp of, their boundaries: the
floor of ``nearest_bev``'s ``limit_period`` and its pi / 4 swap, the direction target's period
and bin, the SmoothL1 knee and the sin difference's zero derivative, and the per-sample GT
capacity.

Referees:

    discrete decisions                 the fp32 restatement (tests/anchor_loss_oracle.py) on
                                       CUDA; its targets are, by construction, what the
                                       reference's fp32 ops give there
    loss values and gradients          the fp64 restatement, as in tests/test_anchor_loss.py
    per-anchor SmoothL1 gradients      the fp32 restatement's autograd on CUDA

Where fp32 and fp64 take different branches at a boundary value, the fp32 referee decides.

CPU tests show that each generator hits the edge it claims, with numpy fp32 arithmetic that forms
``x / period`` as ``x * (1 / period)_f``, as PyTorch does on CUDA (CPU PyTorch divides)."""
import numpy as np
import pytest
import torch

from depth_from_motion_b200 import modules
from depth_from_motion_b200 import synthetic as syn
from tests import anchor_loss_oracle as O
from tests.test_anchor_loss import _check_against_restatement, _check_targets, _kitti_head, \
    _waymo_head

F32 = np.float32
PI_F = F32(np.pi)
INV_PI_F = F32(1) / PI_F
TWO_PI_F = F32(2 * np.pi)
INV_TWO_PI_F = F32(1) / TWO_PI_F
QUARTER_PI_F = F32(np.pi / 4)
HALF_PI_F = F32(np.pi / 2)


def _step(x, n):
    """x moved by n fp32 ulp."""
    x = F32(x)
    to = F32(np.inf) if n > 0 else F32(-np.inf)
    for _ in range(abs(n)):
        x = np.nextafter(x, to)
    return x


def _around(x, k=4):
    return [_step(x, i) for i in range(-k, k + 1)]


# ---- the fp32 period decisions, as the kernel and PyTorch on CUDA form them ----

def _nb_floor(r):
    """floor(r * (1 / pi)_f + 0.5): limit_period's period index in nearest_bev."""
    return float(np.floor(F32(F32(F32(r) * INV_PI_F) + F32(0.5))))


def _nb_swap(r):
    """nearest_bev swaps dx / dy when |r - f pi_f| > (pi / 4)_f."""
    nr = abs(F32(F32(r) - F32(F32(_nb_floor(r)) * PI_F)))
    return bool(nr > QUARTER_PI_F)


def _rot(rg, ra):
    """get_direction_target's rot_gt: the encoded yaw plus the anchor's, in fp32."""
    return F32(F32(F32(rg) - F32(ra)) + F32(ra))


def _dir_floor(rot, off, lim):
    v = F32(F32(rot) - F32(off))
    return float(np.floor(F32(F32(v * INV_TWO_PI_F) + F32(lim))))


def _dir_bin(rot, off, lim):
    v = F32(F32(rot) - F32(off))
    o = F32(v - F32(F32(_dir_floor(rot, off, lim)) * TWO_PI_F))
    return int(min(max(np.floor(F32(o * INV_PI_F)), 0), 1))


def _edge(fn, x0, reach=4096):
    """The fp32 value nearest x0 at which ``fn`` changes: the first value of the upper side."""
    x0 = F32(x0)
    for i in range(reach):
        for x in (_step(x0, i), _step(x0, -i)):
            if fn(_step(x, -1)) != fn(x):
                return x
    raise AssertionError(f'no step of {fn.__name__} within {reach} ulp of {x0}')


RA = (F32(0.0), F32(1.57))   # the anchors' rotations in both configs


def _period_edges(dir_offset, dir_limit_offset):
    """(name, decision function of the GT yaw, boundary yaw) for every period decision in
    [-2 pi, 2 pi]; the direction decisions are taken on an anchor of rotation 0."""
    out = []
    for k in (-1, 0, 1, 2):             # r / pi + 0.5 crosses k
        out.append((f'nb_floor{k}', _nb_floor, _edge(_nb_floor, (k - 0.5) * np.pi)))
    for q in (-7, -5, -3, -1, 1, 3, 5, 7):   # |r - f pi| crosses pi / 4
        out.append((f'nb_swap{q}', _nb_swap, _edge(_nb_swap, q * np.pi / 4)))
    lim = dir_limit_offset
    fl = lambda r: _dir_floor(r, dir_offset, lim)   # noqa: E731
    bn = lambda r: _dir_bin(r, dir_offset, lim)     # noqa: E731
    for m in range(-3, 4):
        r0 = dir_offset + (m - lim) * 2 * np.pi      # (r - off) / 2 pi + lim crosses m
        if abs(r0) <= 2 * np.pi:
            out.append((f'dir_floor{m}', fl, _edge(fl, r0)))
        r1 = dir_offset + (m - lim) * 2 * np.pi + np.pi   # the bin boundary at o = pi
        if abs(r1) <= 2 * np.pi:
            out.append((f'dir_bin{m}', bn, _edge(bn, r1)))
    return out


def _special_yaws():
    """fp32(+-pi / 2) and the LiDAR yaws -ry - pi / 2 of KITTI's ry = 0.00 and +-3.14."""
    out = [HALF_PI_F, -HALF_PI_F]
    for ry in (0.0, 3.14, -3.14):
        out.append(F32(-F32(ry) - HALF_PI_F))
    return out


def _config(head_fn, liga):
    return modules._loss_config(head_fn(), liga)


def _period_yaws(cfg):
    ys = []
    for _, _, b in _period_edges(cfg['dir_offset'], cfg['dir_limit_offset']):
        ys += _around(b)
    for s in _special_yaws():
        ys += _around(s)
    return ys


HEADS = {'kitti': (_kitti_head, True), 'waymo': (_waymo_head, False)}


@pytest.mark.parametrize('config', list(HEADS))
def test_period_sweep_straddles_every_floor(config):
    cfg = _config(*HEADS[config])
    edges = _period_edges(cfg['dir_offset'], cfg['dir_limit_offset'])
    names = {n.rstrip('-0123456789') for n, _, _ in edges}
    assert names == {'nb_floor', 'nb_swap', 'dir_floor', 'dir_bin'}
    for name, fn, b in edges:
        for ra in RA:
            # the decision as the kernel sees it: on the yaw itself for nearest_bev, on the
            # re-added anchor rotation for the direction target
            f = fn if name.startswith('nb') else (lambda r: fn(_rot(r, ra)))  # noqa: E731
            vals = [f(r) for r in _around(b)]
            assert len(set(vals)) == 2, (name, float(b), float(ra), vals)
        assert fn(_step(b, -1)) != fn(b), name
    # ry = 0.00 gives exactly -fp32(pi / 2); the floor of r / pi + 0.5 = 1 steps one ulp below
    # fp32(pi / 2), inside the sweep around it
    assert _special_yaws()[2] == -HALF_PI_F
    assert _edge(_nb_floor, np.pi / 2) == _step(HALF_PI_F, -1)


def _place_gts(anchors, ny, nx, S, R, yaws, labels, spacing, per_sample):
    """GT boxes equal to rotation-0 anchors of size ``labels[i]`` at cells ``spacing`` apart,
    with yaw ``yaws[i]``; ``per_sample`` boxes per sample."""
    an = anchors.reshape(ny, nx, S, R, 7)
    cells = [(y, x) for y in range(spacing // 2, ny, spacing)
             for x in range(spacing // 2, nx, spacing)]
    assert len(cells) >= per_sample
    gts, labs = [], []
    for s0 in range(0, len(yaws), per_sample):
        g = []
        for j, (r, lab) in enumerate(zip(yaws[s0:s0 + per_sample], labels[s0:s0 + per_sample])):
            b = an[cells[j][0], cells[j][1], lab, 0].copy()
            b[6] = r
            g.append(b)
        gts.append(torch.from_numpy(np.stack(g).astype(np.float32)))
        labs.append(torch.tensor(labels[s0:s0 + per_sample], dtype=torch.int64))
    return gts, labs


def _outs(seed, anchors, ny, nx, cfg, B, head_scale=1.0):
    cls, box, dirc, _, _ = syn.make_anchor_loss_case(
        seed, anchors, ny, nx, cfg['num_sizes'], cfg['num_rots'], cfg['num_classes'], [0] * B,
        head_scale=head_scale)
    return [t.cuda().requires_grad_() for t in (cls, box, dirc)]


@pytest.mark.gpu
@pytest.mark.parametrize('config', list(HEADS))
def test_period_edges_match_the_restatement(config):
    make, liga = HEADS[config]
    head = make()
    cfg = modules._loss_config(head, liga)
    ny = nx = 120
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, 'cuda')
    yaws = _period_yaws(cfg)
    labels = [i % cfg['num_sizes'] for i in range(len(yaws))]
    gts, labs = _place_gts(anchors.cpu().numpy(), ny, nx, cfg['num_sizes'], cfg['num_rots'],
                           yaws, labels, spacing=10, per_sample=144)
    B = len(gts)
    outs = _outs(31, anchors.cpu().numpy(), ny, nx, cfg, B)
    _check_against_restatement(f'period_{config}', head, liga, cfg, anchors, outs,
                               [g.cuda() for g in gts], [lab.cuda() for lab in labs],
                               [{} for _ in range(B)])
    # every swept GT got an anchor, so each boundary decided a direction target
    assigned = head._anchor_loss.debug_tensor('assigned_gt')
    for b in range(B):
        got = set(assigned[b].unique().tolist()) - {-1, 0}
        assert got == set(range(1, len(gts[b]) + 1))



# ---- the SmoothL1 knee and the sin difference ----

KNEE_GRID = (24, 24)


def _knee_values(beta):
    b = F32(beta)
    return [b, _step(b, 1), _step(b, -1), F32(0), -b, -_step(b, 1), -_step(b, -1)]


def _yaw_knee(beta):
    """Yaw deltas p whose sin difference against a target of 0, sin(p) cos(0) - cos(p) sin(0) =
    sin(p) (cos(0) = 1 and sin(0) = 0 are exact), is exactly fp32(beta), beta +- 1 ulp, 0 and
    their negatives, with CUDA's fp32 sin.  Then +-fp32(pi / 2), where the derivative
    cos p cos t + sin p sin t vanishes, and +-fp32(pi)."""
    out = []
    for v in _knee_values(beta):
        c = torch.tensor([_step(F32(np.arcsin(float(v))), i) for i in range(-64, 65)],
                         device='cuda')
        hit = torch.nonzero(torch.sin(c) == float(v)).reshape(-1)
        assert len(hit), float(v)
        out.append(F32(c[hit[0]].item()))
    return out + [HALF_PI_F, -HALF_PI_F, PI_F, -PI_F]


def _knee_rows(beta, yaws):
    """Box deltas of the positives, each on a GT equal to its anchor (every target 0): d =
    pred - target is exactly fp32(beta), beta +- 1 ulp, 0 and their negatives on channels 0-5,
    and on the yaw channel the sin differences ``yaws`` give."""
    rows = []
    for k in range(6):
        for d in _knee_values(beta):
            r = np.zeros(7, np.float32)
            r[k] = d
            rows.append(r)
    for y in yaws:
        r = np.zeros(7, np.float32)
        r[6] = y
        rows.append(r)
    return rows


@pytest.mark.parametrize('config', list(HEADS))
def test_knee_targets_are_zero_on_every_grid_anchor(config):
    # a GT equal to its anchor encodes to exactly 0 on every channel (x - x = 0, log(w / w) =
    # log(1) = 0), so the knee rows' deltas are the SmoothL1 arguments themselves
    make, liga = HEADS[config]
    head = make()
    an = modules.grid_anchors(head.extra_cfg['anchor_generator'], *KNEE_GRID, 'cpu')
    assert torch.equal(O.encode(an, an), torch.zeros_like(an))
    assert all(_bits(F32(v) - F32(0)) == _bits(v) for v in _knee_values(_config(make, liga)['beta']))


def _bits(v):
    return np.asarray(v, np.float32).view(np.int32)


def _planted(config, rows, grid, drop_iou, seed):
    """A head, its config, anchors and (cls, box, dirc, gts, labels) with one GT equal to a
    rotation-0 anchor per row, at every other cell, and the row as that anchor's box deltas."""
    make, liga = HEADS[config]
    head = make()
    if drop_iou:
        head.extra_cfg.pop('loss_iou', None)
    cfg = modules._loss_config(head, liga)
    ny, nx = grid
    S, R = cfg['num_sizes'], cfg['num_rots']
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, 'cuda')
    labels = [i % S for i in range(len(rows))]
    gts, labs = _place_gts(anchors.cpu().numpy(), ny, nx, S, R, [F32(0)] * len(rows), labels,
                           spacing=2, per_sample=len(rows))
    cls, box, dirc = (t.detach() for t in _outs(seed, anchors.cpu().numpy(), ny, nx, cfg, 1))
    bv = box.view(1, S, R, 7, ny, nx)
    cells = [(y, x) for y in range(1, ny, 2) for x in range(1, nx, 2)]
    for (y, x), lab, r in zip(cells, labels, rows):
        bv[0, lab, 0, :, y, x] = torch.from_numpy(np.asarray(r, np.float32))
    return head, liga, cfg, anchors, (cls, box, dirc), [g.cuda() for g in gts], \
        [lab.cuda() for lab in labs], cells, labels


@pytest.mark.gpu
@pytest.mark.parametrize('config', list(HEADS))
def test_smooth_l1_knee_and_sin_difference(config):
    cfg0 = _config(*HEADS[config])
    rows = _knee_rows(cfg0['beta'], _yaw_knee(cfg0['beta']))
    # without LIGA's IoU term: the zero rows and yaw +-pi put prediction and target on the same
    # rectangle, a kink of 1 - IoU that the IoU family below referees
    head, liga, cfg, anchors, (cls, box, dirc), gts, labs, cells, labels = _planted(
        config, rows, KNEE_GRID, True, 41)
    S, R = cfg['num_sizes'], cfg['num_rots']
    ny, nx = KNEE_GRID
    outs = [t.clone().requires_grad_() for t in (cls, box, dirc)]
    _check_against_restatement(f'knee_{config}', head, liga, cfg, anchors, outs, gts, labs, [{}])
    # the per-anchor gradient the kernel stores for the SmoothL1 sum, before any normaliser,
    # against the fp32 restatement's autograd of that sum on the same device.  Both form the
    # same fp32 ops (CUDA's sinf / cosf, * (1 / beta)_f, the two sin-difference paths summed
    # last), so 2 ulp leaves room for one rounding on each side
    helper = head._anchor_loss
    g_box = torch.empty_like(box)
    helper.forward(cls, box, dirc, None, g_box, None, None)
    tg = O.targets(anchors, S, R, gts, labs, cfg)
    lab_all = torch.cat([t['labels'] for t in tg])
    pos = torch.nonzero((lab_all >= 0) & (lab_all < cfg['num_classes'])).reshape(-1)
    bf = box.permute(0, 2, 3, 1).reshape(-1, 7).clone().requires_grad_()
    btg = torch.cat([t['bbox_targets'] for t in tg])
    O.smooth_l1_terms(bf[pos], btg[pos], cfg).sum().backward()
    want = bf.grad
    got = g_box.permute(0, 2, 3, 1).reshape(-1, 7)
    ulp = torch.abs(torch.nextafter(want, torch.full_like(want, np.inf)) - want)
    bad = torch.abs(got - want) > 2 * ulp
    assert not bool(bad.any()), (got[bad][:8].tolist(), want[bad][:8].tolist())
    # every planted row is a positive at its anchor, so each edge reached the loss
    asg = helper.debug_tensor('assigned_gt')[0].view(ny, nx, S, R)
    for j, ((y, x), lab) in enumerate(zip(cells, labels)):
        assert int(asg[y, x, lab, 0]) == j + 1


# ---- saturated head outputs ----

@pytest.mark.gpu
@pytest.mark.parametrize('head_scale', [8.0, 30.0])
@pytest.mark.parametrize('config', list(HEADS))
def test_saturated_head_outputs(config, head_scale):
    """make_anchor_loss_case at head_scale 8 and 30: logits far past where the fp32 sigmoid
    rounds to 1 (and, at 30, to 0: both FLT_MIN clamps active), direction-logit gaps near 100.  There the
    fp32 and fp64 focal losses part ways (fp32 clamps log(1 - p) at log(FLT_MIN) once p rounds
    to 1), so loss_cls is refereed by the fp32 restatement's per-logit terms summed in fp64;
    the other terms and all gradients by fp64 as in tests/test_anchor_loss.py."""
    make, liga = HEADS[config]
    head = make()
    cfg = modules._loss_config(head, liga)
    ny, nx, ngt, kw = (64, 60, [20], {}) if liga else (60, 44, [60], dict(cross_class=True))
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, 'cuda')
    cls, box, dirc, gts, labels = syn.make_anchor_loss_case(
        53, anchors.cpu().numpy(), ny, nx, cfg['num_sizes'], cfg['num_rots'],
        cfg['num_classes'], ngt, head_scale=head_scale, **kw)
    outs = [t.cuda().requires_grad_() for t in (cls, box, dirc)]
    gts = [g.cuda() for g in gts]
    labels = [lab.cuda() for lab in labels]
    got = head.loss([outs[0]], [outs[1]], [outs[2]], gts, labels, [{}])
    keys = ['loss_cls', 'loss_bbox', 'loss_dir'] + (['loss_iou'] if cfg['with_iou'] else [])
    W = (0.7, 1.3, 0.9, 1.1)
    sum(w * got[k][0] for w, k in zip(W, keys)).backward()
    tg = O.targets(anchors, cfg['num_sizes'], cfg['num_rots'], gts, labels, cfg)
    _check_targets(head._anchor_loss, tg)
    C = cfg['num_classes']
    x = outs[0].detach().permute(0, 2, 3, 1).reshape(-1, C)
    lab = torch.cat([t['labels'] for t in tg])
    lw = torch.cat([t['label_weights'] for t in tg])
    sat = torch.sigmoid(x)
    assert bool(((sat == 1) & (lab[:, None] != torch.arange(C, device='cuda'))).any())
    # exp(-x) overflows, so p = 0 and log(p) is clamped, only past x = -88: at head_scale 30
    assert bool((sat == 0).any()) == (head_scale > 20)
    terms = (O.sigmoid_focal_loss(x, lab, cfg['gamma'], cfg['alpha']) * lw[:, None]).double()
    n_total = sum(max(t['num_pos'], 1) for t in tg)
    den = (n_total + cfg['normalizer_clamp_value'] if liga else n_total) + O.FLT_EPS
    want_cls = cfg['loss_weight'][0] * terms.sum().item() / den
    # per logit the kernel and the restatement run the same fp32 ops but powf(q, 2) for q * q
    # (a few ulp); a sum of same-signed terms keeps that relative bound, 1e-6 covers it
    assert got['loss_cls'][0].item() == pytest.approx(want_cls, rel=1e-6)
    ins = [t.detach().double().requires_grad_() for t in outs]
    ref = O.losses(*ins, tg, anchors, cfg)
    for k in keys[1:]:
        assert got[k][0].item() == pytest.approx(ref[k].item(), rel=1e-6, abs=1e-12), k
    sum(w * ref[k] for w, k in zip(W, keys)).backward()
    for o, r, nm in zip(outs, ins, ('cls', 'bbox', 'dir')):
        torch.testing.assert_close(o.grad.double(), r.grad, rtol=1e-5, atol=1e-7,
                                   msg=lambda m: f'{config} x{head_scale} grad {nm}: {m}')


# ---- the per-sample GT capacity ----

@pytest.mark.gpu
def test_gt_capacity_of_1024_per_sample():
    head = _waymo_head()
    cfg = modules._loss_config(head, False)
    ny, nx = 60, 44
    anchors = modules.grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, 'cuda')
    cls, box, dirc, gts, labels = syn.make_anchor_loss_case(
        43, anchors.cpu().numpy(), ny, nx, cfg['num_sizes'], cfg['num_rots'],
        cfg['num_classes'], [1024], cross_class=True)
    outs = [t.cuda().requires_grad_() for t in (cls, box, dirc)]
    gts = [g.cuda() for g in gts]
    labels = [lab.cuda() for lab in labels]
    _check_against_restatement('capacity_1024', head, False, cfg, anchors, outs, gts, labels,
                               [{}])
    helper = head._anchor_loss
    before = {k: helper.debug_tensor(k).clone() for k in ('assigned_gt', 'labels')}
    more = [torch.cat([gts[0], gts[0][:1]])]
    with pytest.raises(RuntimeError, match='at most 1024 boxes'):
        head.loss([outs[0]], [outs[1]], [outs[2]], more,
                  [torch.cat([labels[0], labels[0][:1]])], [{}])
    # refused on the host: nothing was launched, the last call's targets stand
    for k, v in before.items():
        assert torch.equal(helper.debug_tensor(k), v), k
