"""fp64 reference detectors for ``test_detector_reference.py``: DfM (KITTI) and MultiViewDfM
(Waymo) composed from the per-stage restatements the stage tests pin to reference fixtures, from
uint8 images to the head outputs and ``get_bboxes_single``'s boxes.

Nothing here calls the CUDA mirrors or the library's metadata code: the metas are rebuilt from
the raw inputs, the parameters come from the detector's state_dict through ``split_state``, and
the glue between the restatements follows the reference detectors line by line
(detectors/dfm.py:264-298, :416-441; detectors/multiview_dfm.py:67-117, :119-209, :321-341).

Feature arithmetic runs in the dtype of the parameters (fp64 in the tests).  Sampling geometry
(plane-sweep grid, frustum grid, projected voxel centres) stays in the reference's fp32, as the
reference computes it from fp32 tensors: the valid masks and the lift's nearest taps are
discontinuous in it, so an fp64 geometry would answer a different question than the reference.

``DEFECTS`` names join mistakes the glue can be told to make, to show that the comparisons in
the tests notice each one.
"""
import math

import numpy as np
import torch

from oracle import dfm_oracle as O
from tests import box_post_oracle as BP
from tests.test_anchor3d_head import anchor3d_head_forward
from tests.test_fpn import fpn_forward
from tests.test_image_prep import prep_reference
from tests.test_liga_resnet import liga_resnet_forward
from tests.test_resnet101 import resnet101_forward
from tests.test_spp_neck import spp_unet_neck_forward

KITTI_STAGES = (('backbone.', 'backbone'), ('neck.', 'neck'),
                ('backbone_stereo.', 'backbone_stereo'),
                ('feature_transformation.', 'feature_transformation'),
                ('backbone_3d.', 'backbone_3d'), ('bbox_head_3d.', 'bbox_head_3d'))
WAYMO_STAGES = (('backbone.', 'backbone'), ('neck.', 'neck'), ('neck_3d.', 'neck_3d'),
                ('bbox_head_3d.', 'bbox_head_3d'))
KITTI_DEFECTS = ('crop_offset_plus_1', 'cur_prev_swapped', 'cur2prev_inverted',
                 'height_compression_nz_c')
WAYMO_DEFECTS = ('scale_factor_one', 'lidar2img_views_permuted', 'fpn_level_1')
DEFECTS = KITTI_DEFECTS + WAYMO_DEFECTS


# ---------------------------------------------------------------------------------------------
# parameters
# ---------------------------------------------------------------------------------------------
class Params(dict):
    """A restatement's parameters; remembers which keys were read."""

    def __init__(self, *args):
        super().__init__(*args)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


def split_state(state, stages, dtype=torch.float64, device='cpu'):
    """The detector state_dict -> one ``Params`` per restatement, keyed by the restatement's own
    names (the module prefix dropped).  A key that maps onto no restatement or onto more than
    one is an error; BatchNorm's ``num_batches_tracked`` is not a parameter of the forward."""
    out = {name: Params() for _, name in stages}
    for k, v in state.items():
        if k.endswith('num_batches_tracked'):
            continue
        hits = [(pre, name) for pre, name in stages if k.startswith(pre)]
        if len(hits) != 1:
            raise KeyError(f'state_dict key {k!r} maps onto {len(hits)} restatements')
        pre, name = hits[0]
        out[name][k[len(pre):]] = v.to(device, dtype)
    return out


def unread(params):
    """Keys no restatement read (after a forward): each one is a parameter the reference
    detector would have used and this composition did not."""
    return sorted(f'{name}.{k}' for name, p in params.items() for k in p if k not in p.read)


# ---------------------------------------------------------------------------------------------
# metas, rebuilt from the raw inputs
# ---------------------------------------------------------------------------------------------
def _padded(n, divisor):
    return -(-n // divisor) * divisor


def kitti_metas(hw, cam2img, cur2prevs, crop_size=(320, 1280), rel_offset_h=(1, 1),
                rel_offset_w=(0.5, 0.5), divisor=32):
    """The img_meta of one KITTI sample after the test pipeline (configs/dfm/dfm_r34_1x8_kitti-
    3d-3class.py:316-338): RandomCrop3D._crop_data (transforms_3d.py:2530-2540) with the
    shipped one-value offset ranges, its intrinsics (:2583-2592), Pad (size_divisor 32), and
    DfMBackbone's view of it (ori_cam2img, ori_shape, no flip, no rescale)."""
    h, w = hw
    margin_h, margin_w = max(h - crop_size[0], 0), max(w - crop_size[1], 0)
    offs = []
    for (lo, hi), margin in ((rel_offset_h, margin_h), (rel_offset_w, margin_w)):
        # randint(lo * margin, hi * margin + 1) has one value when it is an integer
        assert lo == hi and float(lo * margin).is_integer(), (lo, hi, margin)
        offs.append(int(lo * margin))
    y1, x1 = offs
    ch, cw = min(crop_size[0], h), min(crop_size[1], w)
    P = np.array(cam2img, dtype=np.float64)
    K = P[:3, :3].copy()
    T = np.linalg.inv(K) @ P[:3]
    K[0, 2] -= x1
    K[1, 2] -= y1
    cropped = P.copy()
    cropped[:3] = K @ T
    return dict(ori_cam2img=np.array(cam2img, dtype=np.float64), cam2img=cropped,
                cur2prevs=np.asarray(cur2prevs, dtype=np.float64), ori_shape=(h, w, 3),
                img_shape=(ch, cw, 3), pad_shape=(_padded(ch, divisor), _padded(cw, divisor), 3),
                crop_offset=[x1, y1], flip=False, scale_factor=[1.0] * 4)


def waymo_metas(hw, lidar2img, num_views, num_ref_frames, img_scale=(1248, 832), divisor=32):
    """The img_meta of one Waymo sample after the test pipeline: MultiViewImageResize3D with
    keep_ratio (mmcv.rescale_size: s = min(long / max(h, w), short / min(h, w)), new size
    int(x * s + 0.5), factor = new / old per axis in fp32; transforms_3d.py:2409-2434),
    MultiViewImagePad (size_divisor 32); ``input_shape`` as MultiViewDfM.extract_feat sets it
    (multiview_dfm.py:86-89)."""
    h, w = hw
    n = len(lidar2img)
    s = min(max(img_scale) / max(h, w), min(img_scale) / min(h, w))
    nh, nw = int(h * s + 0.5), int(w * s + 0.5)
    ph, pw = _padded(nh, divisor), _padded(nw, divisor)
    return dict(ori_lidar2img=np.asarray(lidar2img, dtype=np.float64),
                scale_factor=np.array([nw / w, nh / h] * 2, dtype=np.float32),
                ori_shape=[(h, w, 3)] * n, img_shape=[(nh, nw, 3)] * n,
                pad_shape=[(ph, pw, 3)] * n, input_shape=(ph, pw),
                num_views=num_views, num_ref_frames=num_ref_frames)


# ---------------------------------------------------------------------------------------------
# anchors
# ---------------------------------------------------------------------------------------------
def anchors(generator, ny, nx):
    """``grid_anchors([[ny, nx]])[0].reshape(-1, 7)`` of Anchor3DRangeGenerator /
    AlignedAnchor3DRangeGenerator (core/anchor/anchor_3d_generator.py:155-220, 255-340, one
    size per range): fp32 linspace centres (aligned: n + 1 points shifted by half a cell),
    rows ordered (y, x, range, rotation)."""
    aligned = generator['type'] == 'AlignedAnchor3DRangeGenerator'
    sizes = generator['sizes']
    ranges = generator['ranges'] * (len(sizes) if len(generator['ranges']) == 1 else 1)
    rots = torch.tensor(generator['rotations'])
    per = []
    for rng, size in zip(ranges, sizes):
        r = torch.tensor(rng)
        cs = []
        for lo, hi, n in ((r[2], r[5], 1), (r[1], r[4], ny), (r[0], r[3], nx)):
            c = torch.linspace(lo, hi, n + aligned)
            if aligned:
                c += (c[1] - c[0]) / 2
            cs.append(c[:n])
        z, y, x = cs
        t = torch.zeros(ny, nx, len(rots), 7)
        t[..., 0] = x.view(1, nx, 1)
        t[..., 1] = y.view(ny, 1, 1)
        t[..., 2] = z[0]
        t[..., 3:6] = torch.tensor(size)
        t[..., 6] = rots
        per.append(t)
    return torch.stack(per, 2).reshape(-1, 7)


def voxel_points(n_voxels, voxel_range):
    """MultiViewDfM's lifting points (multiview_dfm.py:122-123): the aligned generator's
    centres over ``n_voxels`` in fp32, z-major, then y, x fastest."""
    r = torch.tensor(voxel_range)
    cs = []
    for lo, hi, n in ((r[0], r[3], n_voxels[0]), (r[1], r[4], n_voxels[1]),
                      (r[2], r[5], n_voxels[2])):
        c = torch.linspace(lo, hi, n + 1)
        cs.append((c + (c[1] - c[0]) / 2)[:n])
    zz, yy, xx = torch.meshgrid(cs[2], cs[1], cs[0], indexing='ij')
    return torch.stack([xx, yy, zz], -1).reshape(-1, 3)


# ---------------------------------------------------------------------------------------------
# the detectors
# ---------------------------------------------------------------------------------------------
def kitti_forward(params, model, cur, prev, meta, crop_size=(320, 1280), defect=None):
    """DfM.simple_test (dfm.py:416-432 with extract_feat :264-298) of one sample up to the
    head outputs.  cur / prev: uint8 H x W x 3 BGR; meta: ``kitti_metas``.  Returns the joins."""
    p = params
    dt = next(iter(p['backbone'].values())).dtype
    dev = next(iter(p['backbone'].values())).device
    meta = dict(meta)
    if defect == 'crop_offset_plus_1':
        meta['crop_offset'] = [meta['crop_offset'][0], meta['crop_offset'][1] + 1]
    if defect == 'cur2prev_inverted':
        meta['cur2prevs'] = np.linalg.inv(meta['cur2prevs'])
    pair = [cur, prev] if defect != 'cur_prev_swapped' else [prev, cur]
    img, hw = prep_reference(np.stack(pair), 'crop', crop_size, False)
    assert (hw[0], hw[1], 3) == tuple(meta['img_shape'])
    img = img.to(dev, dt)
    cur_imgs, prev_imgs = img[0:1], img[1:2]                                   # :277-278
    cur_feats = [cur_imgs] + list(liga_resnet_forward(p['backbone'], cur_imgs))   # :280-281
    prev_feats = [prev_imgs] + list(liga_resnet_forward(p['backbone'], prev_imgs))
    cur_stereo, cur_sem = spp_unet_neck_forward(p['neck'], cur_feats)        # :285
    prev_stereo, _ = spp_unet_neck_forward(p['neck'], prev_feats)
    # :288-293: cur2prevs becomes a tensor of the image dtype (fp32 in the reference)
    bmeta = dict(ori_cam2img=meta['ori_cam2img'].tolist(),
                 cur2prevs=torch.tensor(meta['cur2prevs'], dtype=torch.float32),
                 ori_shape=meta['ori_shape'], crop_offset=meta['crop_offset'],
                 flip=meta['flip'], scale_factor=meta['scale_factor'])
    depth_cfg = model['depth_cfg']
    bs = model['backbone_stereo']
    cost, stereo, _ = O.dfm_backbone_forward(
        p['backbone_stereo'], cur_stereo, prev_stereo, [bmeta], depth_cfg,
        in_channels=bs['in_channels'], cost_sample_factor=bs['cost_sample_factor'])
    # DepthHead (dfm.py:420-421), its depth samples and factor injected at :322-324
    _, softmax, depth_preds = O.depth_head_forward(
        cost, O.depth_samples(depth_cfg).to(dev, dt), depth_cfg['downsample_factor'])
    ft = model['feature_transformation']
    volume = O.frustum_to_voxel_forward(
        p['feature_transformation'], stereo, softmax,
        [dict(cam2img=meta['cam2img'], pad_shape=meta['pad_shape'])], cur_sem,
        O.frustum_coordinates_3d(model['voxel_cfg']), depth_cfg,
        sem_atten_feat=ft['sem_atten_feat'], stereo_atten_feat=ft['stereo_atten_feat'],
        cat_img_feature=model['neck']['cat_img_feature'], num_3dconvs=ft['num_3dconvs'])
    _, cv, nz, ny, nx = volume.shape                                           # :426-428
    if defect == 'height_compression_nz_c':
        bev_in = volume.transpose(1, 2).reshape(-1, cv * nz, ny, nx)
    else:
        bev_in = volume.view(-1, cv * nz, ny, nx)
    _, bev = O.bev_hourglass_forward(p['backbone_3d'], bev_in)                # :429
    cls, box, dirc = O.liga_anchor3d_head_forward(p['bbox_head_3d'], bev,
                                                  model['bbox_head_3d']['num_convs'])
    return dict(img=cur_imgs, img_feat=cur_feats[-1], stereo_in=cur_stereo, sem=cur_sem,
                cost=cost, stereo=stereo, depth_preds=depth_preds, volume=volume, bev=bev,
                cls=cls, box=box, dir=dirc)


def waymo_forward(params, model, views, meta, img_scale=(1248, 832), defect=None):
    """MultiViewDfM.simple_test (multiview_dfm.py:321-341 with extract_feat :67-117 and
    feature_transformation :119-268) of one sample up to the head outputs.  views: uint8
    H x W x 3 BGR, current frame's cameras first; meta: ``waymo_metas``."""
    p = params
    dt = next(iter(p['backbone'].values())).dtype
    dev = next(iter(p['backbone'].values())).device
    nv, t = meta['num_views'], meta['num_ref_frames'] + 1
    img, _ = prep_reference(np.stack(views), 'rescale', img_scale, True)
    assert tuple(img.shape[-2:]) == tuple(meta['input_shape'])
    level = 1 if defect == 'fpn_level_1' else 0
    feats = []
    for v in range(img.shape[0]):        # one view at a time: the fp64 DCN gather is large
        x = img[v:v + 1].to(dev, dt)
        feats.append(fpn_forward(p['neck'], list(resnet101_forward(p['backbone'], x)))[level])
    feats = torch.cat(feats)
    # feature_transformation (:121-209) on the CPU: the fp32 projection is the CPU GEMM's
    points = voxel_points(model_n_voxels(model), model['anchor_generator']['ranges'][0])
    l2i = [torch.tensor(m, dtype=torch.float32) for m in meta['ori_lidar2img']]
    if defect == 'lidar2img_views_permuted':
        l2i = [l2i[f * nv + (v + 1) % nv] for f in range(t) for v in range(nv)]
    sf = torch.tensor(meta['scale_factor'][:2])                               # :129-136
    if defect == 'scale_factor_one':
        sf = torch.ones(2)
    volume = O.multiview_lift(feats.cpu(), points, model_n_voxels(model), l2i, nv, t, sf, 0,
                              False, meta['input_shape'], meta['img_shape'],
                              model.get('temporal_aggregate', 'mean'))[None].to(dev)
    if model['neck_3d']['type'] == 'DfMNeck':
        bev = O.dfm_neck_forward(p['neck_3d'], volume, model['neck_3d']['in_channels'])[0]
    else:
        bev = O.imvoxel_neck_forward(p['neck_3d'], volume)[0]
    cls, box, dirc = anchor3d_head_forward(p['bbox_head_3d'], bev)
    return dict(img=img, feat=feats, volume=volume, bev=bev, cls=cls, box=box, dir=dirc)


def model_n_voxels(model):
    """MultiViewDfM.__init__ (multiview_dfm.py:54-61): voxels per axis over the first range."""
    r, vs = model['anchor_generator']['ranges'][0], model['voxel_size']
    return [round((r[3 + a] - r[a]) / vs[a]) for a in range(3)]


def boxes(model, cls, box, dirc):
    """get_bboxes_single (anchor3d_head.py:459-547) of one sample's head outputs [C, H, W],
    with the head's anchors, test_cfg and dir offsets."""
    head = model['bbox_head_3d']
    table = anchors(head['anchor_generator'], cls.shape[-2], cls.shape[-1]).to(cls)
    return BP.get_bboxes_single(cls, box, dirc, table, model['test_cfg'], head['num_classes'],
                                True, head.get('dir_offset', -np.pi / 2),
                                head.get('dir_limit_offset', 0.0))


# ---------------------------------------------------------------------------------------------
# box comparison
# ---------------------------------------------------------------------------------------------
IOU_TOL = 0.01        # BEV IoU within this of nms_thr: the suppression decision is ambiguous
MAX_EXEMPT = 0.05     # at most this fraction of the boxes may be exempt


def compare_boxes(got, model, cls, box, dirc, e_cls, e_box, e_dir):
    """Matches the boxes of one sample, ``got`` = (boxes [K, 7], scores, labels) of the library,
    against ``get_bboxes_single`` on the fp64 head outputs (cls, box, dirc [C, H, W]), whose
    absolute errors are bounded by e_cls, e_box, e_dir.

    Every box is identified by its anchor: a got box is the anchor of its label whose fp64
    decode and score it matches within the propagated bounds (score: e_cls / 4, the sigmoid's
    largest slope; box: x, y within e_box * the anchor diagonal, z and sizes within e_box
    times the sizes, yaw within e_box modulo pi).  An anchor kept on both sides must agree in
    score and box, and in yaw up to the pi flip, which only a dir-logit pair within 2 e_dir may
    take.  An anchor kept on one side only must be ambiguous: its score within the bound of
    score_thr or of the nms_pre / max_num cut scores, or a BEV IoU within IOU_TOL of nms_thr
    with a kept box of its class that scores higher (within the score bound), or a suppressor
    that is itself kept on one side only.  Two library boxes on one anchor are a failure.  A
    yaw pi apart with the same direction label is allowed where the decoded yaw lies within the
    yaw bound of limit_period's boundary (yaw - dir_offset = k pi).  Returns dict(matched,
    exempt, failures, total, dir_margins), dir_margins = |dir0 - dir1| of the reference's kept
    anchors."""
    cfg, head = model['test_cfg'], model['bbox_head_3d']
    nc = head['num_classes']
    dir_offset = head.get('dir_offset', -np.pi / 2)
    dir_limit_offset = head.get('dir_limit_offset', 0.0)
    table = anchors(head['anchor_generator'], cls.shape[-2], cls.shape[-1]).double()
    cls, box, dirc = cls.double().cpu(), box.double().cpu(), dirc.double().cpu()
    ref = boxes(model, cls, box, dirc)
    scores = cls.permute(1, 2, 0).reshape(-1, nc).sigmoid()
    deltas = box.permute(1, 2, 0).reshape(-1, 7)
    dirs = dirc.permute(1, 2, 0).reshape(-1, 2)
    dec = BP.decode(table, deltas)
    ds = e_cls / 4 + 1e-6
    diag = torch.sqrt(table[:, 3] ** 2 + table[:, 4] ** 2)
    tol = torch.stack([diag, diag, table[:, 5] + dec[:, 5], dec[:, 3], dec[:, 4], dec[:, 5]],
                      -1) * (2 * e_box) + 1e-4
    yaw_tol = 2 * e_box + 1e-4
    thr, nms_thr = cfg['score_thr'], cfg['nms_thr']
    # scores at the nms_pre and max_num cuts
    maxs = scores.max(1)[0]
    pre_cut = float(maxs.sort(descending=True)[0][cfg['nms_pre'] - 1]) \
        if 0 < cfg['nms_pre'] < maxs.numel() else None
    final = torch.sort(ref['scores'], descending=True)[0]
    num_cut = float(final[cfg['max_num'] - 1]) if final.numel() >= cfg['max_num'] else None

    def yaw_diff(a, b, period=math.pi):
        d = (a - b) % period
        return min(d, period - d)

    def at_period_boundary(a):
        # limit_period(yaw - dir_offset, dir_limit_offset, pi) (anchor3d_head.py:541-545)
        v = (float(dec[a, 6]) - dir_offset) / math.pi + dir_limit_offset
        return abs(v - round(v)) * math.pi <= yaw_tol

    def box_close(a, g):
        return bool(((dec[a, :6] - g[:6]).abs() <= tol[a]).all()) and \
            yaw_diff(float(dec[a, 6]), float(g[6])) <= yaw_tol

    ref_boxes, ref_labels = ref["boxes"], ref["labels"]
    ref_keep = {c: [int(a) for a in ref['keep'][c]] for c in range(nc)}
    if ref_boxes.shape[0] < sum(len(v) for v in ref_keep.values()):      # max_num cut
        kept_scores = torch.cat([scores[torch.tensor(ref_keep[c], dtype=torch.long), c]
                                 for c in range(nc)])
        inds = torch.argsort(kept_scores, descending=True, stable=True)[:cfg['max_num']]
        flat = [(c, a) for c in range(nc) for a in ref_keep[c]]
        ref_keep = {c: [] for c in range(nc)}
        for i in inds.tolist():
            ref_keep[flat[i][0]].append(flat[i][1])
    gb, gs, gl = (x.double().cpu() for x in got)
    failures, matched, exempt, margins = [], 0, 0, []
    for c in range(nc):
        rk = set(ref_keep[c])
        sel = torch.nonzero(gl == c).flatten().tolist()
        got_anchor = {}
        for i in sel:
            near = torch.nonzero((scores[:, c] - gs[i]).abs() <= ds).flatten()
            hit = [int(a) for a in near if box_close(int(a), gb[i])]
            if not hit:
                failures.append(f'class {c}: library box {i} (score {float(gs[i]):.5f}) '
                                f'matches no anchor')
                continue
            hit.sort(key=lambda a: (a not in rk, float((dec[a, :6] - gb[i, :6]).abs().sum())))
            if hit[0] in got_anchor:
                failures.append(f'class {c}: library boxes {got_anchor[hit[0]]} and {i} are '
                                f'both anchor {hit[0]}')
                continue
            got_anchor[hit[0]] = i
        gk = set(got_anchor)
        one_sided = rk ^ gk
        kept = rk | gk
        bev = BP.nms_box(dec)

        def ambiguous(a):
            s = float(scores[a, c])
            if abs(s - thr) <= ds:
                return True
            if pre_cut is not None and abs(float(maxs[a]) - pre_cut) <= ds:
                return True
            if num_cut is not None and abs(s - num_cut) <= ds:
                return True
            higher = [b for b in kept if b != a and float(scores[b, c]) >= s - ds]
            if not higher:
                return False
            iou = BP.rotated_iou(bev[a:a + 1], bev[torch.tensor(higher)])
            for b, v in zip(higher, iou.tolist()):
                if abs(v - nms_thr) <= IOU_TOL or (v > nms_thr and b in one_sided):
                    return True
            return False
        margins += [float((dirs[a, 0] - dirs[a, 1]).abs()) for a in sorted(rk)]
        for a in sorted(kept):
            if a in rk and a in gk:
                i = got_anchor[a]
                j = int(torch.nonzero((ref_labels == c) &
                                      (ref_boxes[:, :6] == dec[a, :6]).all(1))[0])
                if abs(float(gs[i] - scores[a, c])) > ds:
                    failures.append(f'class {c} anchor {a}: score {float(gs[i])} vs '
                                    f'{float(scores[a, c])}')
                dyaw = yaw_diff(float(gb[i, 6]), float(ref_boxes[j, 6]), 2 * math.pi)
                if dyaw > yaw_tol and abs(dyaw - math.pi) > yaw_tol:
                    failures.append(f'class {c} anchor {a}: yaw {float(gb[i, 6])} vs '
                                    f'{float(ref_boxes[j, 6])}')
                elif dyaw > yaw_tol and float((dirs[a, 0] - dirs[a, 1]).abs()) > 2 * e_dir \
                        and not at_period_boundary(a):
                    failures.append(f'class {c} anchor {a}: direction flipped with dir logits '
                                    f'{dirs[a].tolist()}')
                matched += 1
            elif ambiguous(a):
                exempt += 1
            else:
                side = 'reference' if a in rk else 'library'
                failures.append(f'class {c} anchor {a}: kept by the {side} only, score '
                                f'{float(scores[a, c]):.5f}, not ambiguous')
    return dict(matched=matched, exempt=exempt, failures=failures,
                total=int(ref_boxes.shape[0]), dir_margins=margins)
