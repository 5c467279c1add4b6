"""The whole detectors, ``modules.DfM`` (KITTI) and ``modules.MultiViewDfM`` (Waymo): built from
the shipped configs, loaded from one checkpoint, and run from decoded images to scored boxes.

CPU: every shipped config builds its detector through ``Config.fromfile`` + ``build_detector``
with the reference constructor's injections; ``checkpoint.load_detector`` loads every inference
key, reports the training-only ones, rejects a stray key and reads LIGA-DfM names.

GPU (full size): ``simple_test`` on images prepared by ``image_prep`` gives the boxes, scores and
labels of the already-tested mirrors chained by hand below, line by line after
detectors/dfm.py:264-298, 416-441 and detectors/multiview_dfm.py:67-117, 321-341; plus the
hand-offs between modules (cur / prev order, Waymo batches, ``pseudo_lidar``, malformed input).
"""
import copy
import gc
import json
import os

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi, checkpoint, image_prep, modules, registry
from depth_from_motion_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CONFIGS = json.load(open(os.path.join(GOLDEN, 'detector_configs.json')))
KITTI = 'dfm_r34_1x8_kitti-3d-3class.py'
CAMSYNC = 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync.py'
SWEEPS10 = 'multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync_10sweeps.py'


def build(name, tmp_path=None):
    """The detector of a shipped config, parsed with Config.fromfile from a flat config file."""
    model = CONFIGS[name]
    if tmp_path is None:
        return registry.build_detector(copy.deepcopy(model))
    path = tmp_path / name
    path.write_text(f'model = {model!r}\n')
    return registry.build_detector(registry.Config.fromfile(str(path)).model)


def random_state(det, seed):
    """Random inference parameters for every key of the detector's state_dict."""
    rng = np.random.RandomState(seed)
    out = {}
    for k, v in det.state_dict().items():
        shape = tuple(v.shape)
        if k.endswith('num_batches_tracked'):
            out[k] = v.clone()
            continue
        if k.endswith('running_var'):
            a = 1 + 0.1 * np.abs(rng.standard_normal(shape))
        elif k.endswith('running_mean') or k.endswith('bias'):
            a = 0.1 * rng.standard_normal(shape)
        elif len(shape) == 1:            # norm weights
            a = 1 + 0.1 * rng.standard_normal(shape)
        else:
            fan_in = int(np.prod(shape[1:]))
            a = rng.standard_normal(shape) / np.sqrt(fan_in)
        out[k] = torch.from_numpy(a.astype(np.float32))
    return out


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_shipped_configs_build_the_detector(name, tmp_path):
    det = build(name, tmp_path)
    model = CONFIGS[name]
    if model['type'] == 'DfM':
        assert type(det) is modules.DfM
        assert isinstance(det.backbone, modules.LIGAResNet)
        assert isinstance(det.neck, modules.SPPUNetNeck)
        assert isinstance(det.backbone_3d, modules.BEVHourglass)
        assert isinstance(det.bbox_head_3d, modules.LIGAAnchor3DHead)
        # injections of dfm.py:43-109
        assert det.backbone_stereo.depth_cfg == model['depth_cfg']
        assert det.backbone_stereo.downsampled_depth.shape == (72,)
        assert float(det.backbone_stereo.downsampled_depth[0]) == pytest.approx(2 + 2 * 0.2)
        assert det.depth_head.depth_samples.shape == (288,)
        assert det.depth_head.downsample_factor == 4
        ft = det.feature_transformation
        assert ft.cat_img_feature and ft.in_sem_channels == 32 and ft.depth_cfg is not None
        assert tuple(ft.coordinates_3d.shape) == (20, 304, 288, 3)
        assert det.bbox_head_3d.normalizer_clamp_value == model['normalizer_clamp_value']
        assert det.bbox_head_3d.test_cfg == model['test_cfg']
        for name_ in ('lidar_model', 'neck_2d', 'bbox_head_2d', 'depth_head_2d'):
            assert not hasattr(det, name_)
    else:
        assert type(det) is modules.MultiViewDfM
        assert isinstance(det.backbone, modules.ResNet) and isinstance(det.neck, modules.FPN)
        assert isinstance(det.neck_3d, (modules.DfMNeck, modules.OutdoorImVoxelNeck))
        assert isinstance(det.bbox_head_3d, modules.Anchor3DHead)
        assert det.n_voxels == [220, 300, 12]
        assert det.voxel_range == model['anchor_generator']['ranges'][0]
        assert det.temporal_aggregate == model.get('temporal_aggregate', 'mean')
        assert not det.with_backbone_3d and not det.with_depth_head
    det.train()
    with pytest.raises(RuntimeError, match='eval'):
        det.simple_test(torch.zeros(1, 2, 3, 32, 32), [{}])


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_the_shipped_config_files_parse_and_build(name):
    """Config.fromfile on the shipped config file itself (its variables and nesting), where the
    reference tree is present; the recorded model dict above is what it parses to."""
    from oracle.ref_loader import REFERENCE_ROOT
    path = os.path.join(REFERENCE_ROOT, 'configs', 'dfm', name)
    if not os.path.isfile(path):
        pytest.skip('the reference configs are not present')
    model = registry.Config.fromfile(path).model
    assert json.loads(json.dumps(dict(model), default=list)) == CONFIGS[name]
    det = registry.build_detector(model)
    assert type(det).__name__ == CONFIGS[name]['type']


def test_dfm_accepts_cur2prevs_as_a_tensor():
    """extract_feat leaves cur2prevs a host fp32 tensor whether the meta holds a list, an array or
    a tensor (the reference's own extract_feat turns it into one on the image's device)."""
    class Call(torch.nn.Module):
        def __init__(self, fn):
            super().__init__()
            self.fn = fn

        def forward(self, *args):
            return self.fn(*args)
    det = build(KITTI).eval()
    seen = []
    det.backbone = Call(lambda x: (x[:, :1],))
    det.neck = Call(lambda feats: (feats[0], feats[0]))
    det.backbone_stereo = Call(lambda c, p, metas: seen.append(metas[0]['cur2prevs']) or (c,) * 3)
    c2p = syn.KITTI_CUR2PREV[2:3]
    for value in (c2p.tolist(), c2p, torch.from_numpy(c2p).float()):
        det.extract_feat(torch.zeros(1, 2, 3, 8, 8), [dict(cur2prevs=value)])
    assert len(seen) == 3
    for got in seen:
        assert got.dtype == torch.float32 and got.device.type == 'cpu'
        assert torch.equal(got, torch.from_numpy(c2p).float())


def test_detectors_are_not_forced_into_mmdet():
    assert 'DfM' in registry.DETECTORS and 'MultiViewDfM' in registry.DETECTORS
    with pytest.raises(AssertionError):
        registry.build_detector(dict(CONFIGS[KITTI]), test_cfg=dict(max_num=1))


def _liga_name(key):
    """The LIGA-DfM release's name of a detector key (convert_dfm_checkpoints.py:34-63 read
    backwards)."""
    rows = (('backbone.', 'backbone_3d.feature_backbone.'),
            ('neck.', 'backbone_3d.feature_neck.'),
            ('feature_transformation.voxel_convs.', 'backbone_3d.rpn3d_convs.'),
            ('backbone_stereo.', 'backbone_3d.'),
            ('backbone_3d.compress_conv.', 'backbone_2d.rpn3d_conv2.'),
            ('backbone_3d.bev_hourglass.', 'backbone_2d.rpn3d_conv3.'),
            ('bbox_head_3d.cls_convs.', 'dense_head.rpn3d_cls_convs.'),
            ('bbox_head_3d.reg_convs.', 'dense_head.rpn3d_bbox_convs.'),
            ('bbox_head_3d.conv_reg.', 'dense_head.conv_box.'),
            ('bbox_head_3d.', 'dense_head.'))
    for new, old in rows:
        if key.startswith(new):
            return old + key[len(new):]
    raise AssertionError(key)


def test_load_detector_on_a_synthetic_checkpoint():
    det = build(KITTI)
    state = random_state(det, 1)
    training = {'lidar_model.backbone.compress_conv.0.weight': torch.zeros(2),
                'neck_2d.fpn_convs.0.conv.weight': torch.zeros(2),
                'bbox_head_2d.conv_cls.weight': torch.zeros(2),
                'conv_imitation.0.weight': torch.zeros(2),
                'norm_imitation.0.weight': torch.zeros(2)}
    skipped = checkpoint.load_detector({'state_dict': {**state, **training}}, det)
    assert skipped == sorted(training)
    got = det.state_dict()
    assert set(got) == set(state) and any(k.startswith('backbone_3d.') for k in got)
    assert all(torch.equal(got[k], v) for k, v in state.items())
    with pytest.raises(KeyError, match='stray'):
        checkpoint.load_detector({**state, 'stray.weight': torch.zeros(1)}, build(KITTI))
    with pytest.raises(RuntimeError, match='Missing'):
        checkpoint.load_detector({k: v for k, v in state.items()
                                  if not k.startswith('backbone_3d.')}, build(KITTI))
    # LIGA-DfM names, as the release stores them
    liga = {_liga_name(k): v for k, v in random_state(det, 2).items()}
    liga['global_step'] = torch.zeros(1)
    liga['lidar_model.backbone_2d.rpn3d_conv2.0.weight'] = torch.zeros(2)
    liga['backbone_3d.sem_neck.x.weight'] = torch.zeros(2)
    liga['dense_head.conv_imitation.0.weight'] = torch.zeros(2)
    fresh = build(KITTI)
    skipped = checkpoint.load_detector({'model_state': liga}, fresh)
    assert skipped == ['conv_imitation.0.weight', 'lidar_model.backbone_2d.rpn3d_conv2.0.weight',
                       'neck_2d.x.weight']
    want = random_state(det, 2)
    got = fresh.state_dict()
    assert all(torch.equal(got[k], v) for k, v in want.items())
    # load_hot_path keeps reading LIGA names as before: dense_head.* is not the 3-D head's
    parts = checkpoint.hot_path_state_dicts({'model_state': liga})
    assert not parts['bbox_head_3d'] and parts['backbone_stereo']


def test_malformed_detector_input_is_refused_before_any_launch():
    det = build(KITTI).eval()
    with pytest.raises(ValueError, match='img must be'):
        det.simple_test(torch.zeros(1, 1, 3, 32, 32), [{}])
    with pytest.raises(ValueError, match='img must be'):
        det.simple_test(torch.zeros(1, 2, 32, 32), [{}])


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _cuda_detector(name, seed):
    _free()
    det = build(name)
    checkpoint.load_detector(random_state(det, seed), det)
    return det.cuda().eval()


def _free(det=None):
    """Destroys the detector's library handles now rather than at garbage collection: a
    full-size ResNet-101 handle holds gigabytes, and the GPU tests share one process."""
    if det is not None:
        for m in det.modules():
            if hasattr(m, 'release'):
                m.release()
            if hasattr(m, '_box_post'):
                m._box_post.release()
    gc.collect()
    torch.cuda.empty_cache()


def _kitti_inputs(seed, swap=False):
    rng = np.random.RandomState(seed)
    # smooth images, so the plane sweep has structure to match
    cur = (127 + 100 * np.tanh(syn.smooth_field(rng, 3, 375, 1242, cell=16)[0].numpy())).astype(
        np.uint8).transpose(1, 2, 0).copy()
    prev = np.roll(cur, 3, axis=1)
    if swap:
        cur, prev = prev, cur
    c2p = syn.KITTI_CUR2PREV[2:3]
    return image_prep.prepare_kitti(cur, [prev], syn.KITTI_P2, c2p)


def _waymo_inputs(seed, num_frames, batch=1):
    rng = np.random.RandomState(seed)
    ori = np.diag([1 / 0.65, 1 / 0.65, 1, 1]) @ syn.waymo_lidar2img(num_frames)
    imgs, metas = [], []
    for _ in range(batch):
        views = [rng.randint(0, 256, (1280, 1920, 3), dtype=np.uint8) for _ in range(5 * num_frames)]
        img, m = image_prep.prepare_waymo(views, ori, num_ref_frames=num_frames - 1)
        imgs.append(img)
        metas += m
    return torch.cat(imgs), metas


def _same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert set(x) == set(y), what
        n = x['boxes_3d'].shape[0]
        print(what, 'sample', i, 'boxes', n, 'vs', y['boxes_3d'].shape[0])
        for k in ('boxes_3d', 'scores_3d', 'labels_3d'):
            assert torch.equal(x[k], y[k]), (what, i, k)


def kitti_by_hand(det, img, img_metas):
    """detectors/dfm.py:416-441 with :264-298, the mirrors called as the reference calls them."""
    img_metas = copy.deepcopy(img_metas)
    cur_imgs = img[:, 0]
    prev_imgs = img[:, 1]
    cur_feats = det.backbone(cur_imgs)
    cur_feats = [cur_imgs] + list(cur_feats)
    prev_feats = det.backbone(prev_imgs)
    prev_feats = [prev_imgs] + list(prev_feats)
    cur_stereo_feat, cur_sem_feat = det.neck(cur_feats)
    prev_stereo_feat, prev_sem_feat = det.neck(prev_feats)
    for img_meta in img_metas:
        img_meta['cur2prevs'] = torch.tensor(np.asarray(img_meta['cur2prevs']), dtype=img.dtype)
    mono_stereo_costs, stereo_feats, mono_feats = det.backbone_stereo(
        cur_stereo_feat, prev_stereo_feat, img_metas)
    # DepthHead fused into FrustumToVoxel, as test_box_regression_parity_end_to_end runs it
    logits = modules.CostLogits(mono_stereo_costs, depth_samples=det.depth_head.depth_samples)
    volume_feat = det.feature_transformation(stereo_feats, logits, img_metas, cur_sem_feat)
    _, Cv, Nz, Ny, Nx = volume_feat.shape
    bev_feat = volume_feat.view(-1, Cv * Nz, Ny, Nx)
    bev_feat_prehg, bev_feat = det.backbone_3d(bev_feat)
    outs = det.bbox_head_3d([bev_feat])
    bbox_list = det.bbox_head_3d.get_bboxes(*outs, img_metas)
    bbox_results = [modules.bbox3d2result(b, s, l) for b, s, l in bbox_list]
    for bbox_result in bbox_results:
        bbox_result['pseudo_lidar'] = True
    return bbox_results


def waymo_by_hand(det, img, img_metas):
    """detectors/multiview_dfm.py:321-341 with :67-117."""
    img_metas = copy.deepcopy(img_metas)
    batch_size, _, C_in, H, W = img.shape
    num_views = img_metas[0]['num_views']
    num_ref_frames = img_metas[0]['num_ref_frames']
    num_frames = num_ref_frames + 1 if num_ref_frames > 0 else 1
    input_shape = img.shape[-2:]
    for img_meta in img_metas:
        img_meta.update(input_shape=input_shape)
    if num_ref_frames > 0:
        cur_imgs = img[:, :num_views].reshape(-1, C_in, H, W)
        prev_imgs = img[:, num_views:].reshape(-1, C_in, H, W)
        cur_feats = det.neck(det.backbone(cur_imgs))[0]
        prev_feats = det.neck(det.backbone(prev_imgs))[0]
        _, C_feat, H_feat, W_feat = cur_feats.shape
        cur_feats = cur_feats.view(batch_size, -1, C_feat, H_feat, W_feat)
        prev_feats = prev_feats.view(batch_size, -1, C_feat, H_feat, W_feat)
        batch_feats = torch.cat([cur_feats, prev_feats], dim=1)
    else:
        batch_feats = det.neck(det.backbone(img.view(-1, C_in, H, W)))[0]
        _, C_feat, H_feat, W_feat = batch_feats.shape
        batch_feats = batch_feats.view(batch_size, -1, C_feat, H_feat, W_feat)
    feats = det.feature_transformation(batch_feats, img_metas, num_views, num_frames)
    outs = det.bbox_head_3d([feats[0]])
    bbox_list = det.bbox_head_3d.get_bboxes(*outs, img_metas)
    return [modules.bbox3d2result(b, s, l) for b, s, l in bbox_list]


@pytest.mark.gpu
def test_kitti_detector_end_to_end():
    det = _cuda_detector(KITTI, 11)
    try:
        _kitti_end_to_end(det)
    finally:
        _free(det)


def _kitti_end_to_end(det):
    img, metas = _kitti_inputs(12)
    assert img.shape == (1, 2, 3, 320, 1248)
    with torch.no_grad():
        got = det.simple_test(img, copy.deepcopy(metas))
        ref = kitti_by_hand(det, img, metas)
        swapped = det.simple_test(*_kitti_inputs(12, swap=True))
    capi.sync_check()
    assert got[0]['pseudo_lidar'] is True
    assert got[0]['boxes_3d'].shape[1] == 7 and got[0]['boxes_3d'].shape[0] > 0
    _same(got, ref, 'kitti')
    assert not (got[0]['boxes_3d'].shape == swapped[0]['boxes_3d'].shape and
                torch.equal(got[0]['boxes_3d'], swapped[0]['boxes_3d'])), 'cur / prev swap'
    # malformed input: refused before any kernel is launched
    launches = capi.launch_counters()[0]
    with pytest.raises(ValueError):
        det.simple_test(img[:, :1], metas)
    with pytest.raises(ValueError):
        det.simple_test(img, metas * 2)
    with pytest.raises(ValueError):
        image_prep.prepare_kitti(np.zeros((375, 1242, 3), np.uint8),
                                 [np.zeros((370, 1242, 3), np.uint8)], syn.KITTI_P2,
                                 syn.KITTI_CUR2PREV[2:3])
    assert capi.launch_counters()[0] == launches


@pytest.mark.gpu
@pytest.mark.parametrize('name,num_frames', [(CAMSYNC, 1), (SWEEPS10, 2)])
def test_waymo_detector_end_to_end(name, num_frames):
    det = _cuda_detector(name, 21)
    try:
        _waymo_end_to_end(det, name, num_frames)
    finally:
        _free(det)


def _waymo_end_to_end(det, name, num_frames):
    img, metas = _waymo_inputs(22, num_frames)
    assert img.shape == (1, 5 * num_frames, 3, 832, 1248)
    with torch.no_grad():
        got = det.simple_test(img, copy.deepcopy(metas))
        ref = waymo_by_hand(det, img, metas)
    capi.sync_check()
    assert 'pseudo_lidar' not in got[0] and got[0]['boxes_3d'].shape[0] > 0
    _same(got, ref, name)
    if num_frames == 2:
        # the previous views are not interchangeable with the current ones
        swapped = torch.cat([img[:, 5:], img[:, :5]], 1)
        with torch.no_grad():
            other = det.simple_test(swapped, copy.deepcopy(metas))
        assert not (other[0]['boxes_3d'].shape == got[0]['boxes_3d'].shape and
                    torch.equal(other[0]['boxes_3d'], got[0]['boxes_3d'])), 'cur / prev swap'
        # B = 2 equals two B = 1 calls
        img2, metas2 = _waymo_inputs(23, num_frames, batch=2)
        with torch.no_grad():
            both = det.simple_test(img2, copy.deepcopy(metas2))
            one = [det.simple_test(img2[b:b + 1], copy.deepcopy(metas2[b:b + 1]))[0]
                   for b in range(2)]
        _same(both, one, 'waymo B=2')
    launches = capi.launch_counters()[0]
    with pytest.raises(ValueError):
        det.simple_test(img[:, :4], metas)
    assert capi.launch_counters()[0] == launches
