"""The contract every parameterised handle of include/dfm_b200.h keeps, checked for each of the
eleven at a small valid size against the state_dict its Python mirror uploads:

- right after create, missing_params counts every key the mirror's _ParamSync uploads
  (num_batches_tracked is skipped);
- an unknown key, or a known key with the wrong element count, returns DFM_ERR_INVALID and
  leaves the key missing;
- a forward with parameters missing returns DFM_ERR_STATE and names a missing key;
- after the whole state_dict is uploaded nothing is missing, and a key can be uploaded again;
- the debug hook refuses an unknown name and a tensor no forward has written, and after a
  forward a size other than what it wrote;
- destroy(NULL) returns DFM_OK.

The handles without parameters (the losses, box_post, kitti_eval) keep the debug-hook and
destroy parts."""
import ctypes

import pytest

from depth_from_motion_b200 import capi, modules
from depth_from_motion_b200 import synthetic as syn

vp = ctypes.c_void_p
ERR_INVALID, ERR_STATE = 1, 3   # DFM_ERR_* of include/dfm_b200.h
FAMILIES = ('backbone', 'neck', 'frustum', 'bev_hourglass', 'anchor_head', 'anchor3d_head',
            'stereo_tail', 'spp_neck', 'fpn', 'liga_resnet', 'resnet101')
GN = dict(type='GN', num_groups=32)


def _uploaded(mirror):
    """(key, fp32 host tensor) pairs in the order _ParamSync uploads them."""
    import torch
    g = torch.Generator().manual_seed(0)
    out = []
    for k, v in mirror.state_dict().items():
        if k.endswith('num_batches_tracked'):
            continue
        t = torch.rand(v.shape, generator=g) + (0.5 if k.endswith('running_var') else -0.5)
        out.append((k, t.float().contiguous()))
    return out


def _create(L, family, *args):
    hd = vp()
    capi.check(getattr(L, f'dfm_{family}_create')(*args, ctypes.byref(hd)),
               f'dfm_{family}_create')
    return hd


def _cases(L, p):
    """(family, handle, mirror, forward of the handle on dummy pointers, debug names:
    (a tensor a forward writes, a name the handle does not know) or None)"""
    from tests.test_anchor3d_head import waymo_head
    from tests.test_fpn import IN_CH, waymo_fpn
    from tests.test_liga_resnet import BACKBONE_CFG as LIGA_CFG
    from tests.test_resnet101 import BACKBONE_CFG as R101_CFG
    from tests.test_spp_neck import NECK_CFG
    four = (vp * 4)(p, p, p, p)
    geom = capi.Geometry()
    cam = (ctypes.c_double * 16)()
    ci = ctypes.c_int * 4
    cases = []

    def add(family, h, mirror, forward, dbg=None):
        cases.append((family, h, mirror, forward, dbg))

    add('backbone', _create(L, 'backbone', ctypes.byref(capi.BackboneDesc(32, 32, 16, 32, 8, 4, 1,
                                                                          0))),
        modules.DfMBackbone(in_channels=32, depth_cfg=syn.depth_cfg_for(8)),
        lambda h: L.dfm_backbone_forward(h, p, p, ctypes.byref(geom), p, p, p, None),
        ('raw0', 'nope'))
    for frames, mirror in ((2, modules.DfMNeck(32, 64, num_frames=2)),
                           (0, modules.OutdoorImVoxelNeck(32, 64))):
        add('neck', _create(L, 'neck', ctypes.byref(capi.NeckDesc(32, 64, frames, 8, 8, 12, 0))),
            mirror, lambda h: L.dfm_neck_forward(h, p, p, None), ('mono.0', 'mono.9'))
    for convs in (1, 4):
        d = capi.FrustumDesc(convs, 32, 32, 32, 1, 0, 1, 8, 8, 8, 8, 8, 4, 8, 8, 8, 2.0, 59.6, 0)
        xs = (ctypes.c_float * 8)()
        hd = vp()
        capi.check(L.dfm_frustum_create(ctypes.byref(d), xs, xs, xs, ctypes.byref(hd)),
                   'dfm_frustum_create')
        add('frustum', hd, modules.FrustumToVoxel(num_3dconvs=convs),
            lambda h: L.dfm_frustum_forward(h, p, 0, None, None, None, None, p, cam, 32, 32, p,
                                            None),
            ('vox', 'conv9'))
    add('bev_hourglass', _create(L, 'bev_hourglass', ctypes.byref(capi.BevDesc(64, 64, 8, 8, 0))),
        modules.BEVHourglass(64, 64, norm_cfg=GN),
        lambda h: L.dfm_bev_hourglass_forward(h, p, p, p, None), ('conv1', 'conv7'))
    for convs, dirs in ((2, True), (0, False)):
        mirror = modules.LIGAAnchor3DHead(num_classes=3, in_channels=64, feat_channels=64,
                                          num_convs=convs, norm_cfg=GN,
                                          use_direction_classifier=dirs,
                                          anchor_generator=syn.KITTI_ANCHOR_GENERATOR)
        desc = capi.AnchorHeadDesc(64, 64, convs, 18, 42, 12 if dirs else 0, 8, 8, 0)
        add('anchor_head', _create(L, 'anchor_head', ctypes.byref(desc)), mirror,
            lambda h: L.dfm_anchor_head_forward(h, p, p, p, p, None), ('cls_out', 'cls4'))
    for dirs in (True, False):
        mirror = waymo_head(in_channels=64, feat_channels=64, use_direction_classifier=dirs)
        desc = capi.Anchor3DHeadDesc(64, 18, 42, 12 if dirs else 0, 8, 8, 0)
        add('anchor3d_head', _create(L, 'anchor3d_head', ctypes.byref(desc)), mirror,
            lambda h: L.dfm_anchor3d_head_forward(h, p, p, p, p, None))
    add('stereo_tail', _create(L, 'stereo_tail', 16, 16, 0), modules.SPPUNetNeckTail(),
        lambda h: L.dfm_stereo_tail_forward(h, p, p, p, None))
    add('spp_neck', _create(L, 'spp_neck', 512, 1024, 0), modules.SPPUNetNeck(**NECK_CFG),
        lambda h: L.dfm_spp_neck_forward(h, p, p, p, p, p, p, p, p, None), ('x0', 'x2'))
    desc = capi.FpnDesc(ci(*IN_CH), 64, ci(8, 4, 2, 1), ci(8, 4, 2, 1), 1, 0)
    add('fpn', _create(L, 'fpn', ctypes.byref(desc)), waymo_fpn(),
        lambda h: L.dfm_fpn_forward(h, four, four, None), ('merged0', 'merged4'))
    add('liga_resnet', _create(L, 'liga_resnet', ctypes.byref(capi.LigaResNetDesc(32, 32, 1, 0))),
        modules.LIGAResNet(**LIGA_CFG),
        lambda h: L.dfm_liga_resnet_forward(h, p, four, None), ('stem', 'pool'))
    add('resnet101', _create(L, 'resnet101', ctypes.byref(capi.ResNet101Desc(64, 64, 1, 0))),
        modules.ResNet(**R101_CFG),
        lambda h: L.dfm_resnet101_forward(h, p, four, None), ('stem', 'layer5.0'))
    return cases


def _debug(L, family, h, name, out, numel):
    return getattr(L, f'dfm_{family}_debug_tensor')(h, name.encode(), out, numel, None)


def _error():
    return capi.lib().dfm_last_error().decode()


@pytest.mark.gpu
def test_handle_contract():
    import torch
    L = capi.lib()
    buf = torch.zeros(1 << 16, device='cuda')
    p = vp(buf.data_ptr())
    seen = set()
    for family, h, mirror, forward, dbg in _cases(L, p):
        seen.add(family)
        try:
            count = getattr(L, f'dfm_{family}_missing_params')
            set_param = getattr(L, f'dfm_{family}_set_param')

            def put(key, t, numel=None):
                return set_param(h, key.encode(), vp(t.data_ptr()),
                                 t.numel() if numel is None else numel)

            params = _uploaded(mirror)
            n = len(params)
            assert count(h) == n, family
            one = torch.zeros(1)
            assert put('no.such.key', one) == ERR_INVALID, family
            assert count(h) == n, family
            key, t = params[0]
            bigger = torch.zeros(t.numel() + 1)
            assert put(key, bigger) == ERR_INVALID, (family, key)
            assert 'element' in _error() or 'expected' in _error(), (family, _error())
            assert count(h) == n, family
            assert forward(h) == ERR_STATE, family
            assert 'missing parameter' in _error(), family
            if dbg:
                assert _debug(L, family, h, dbg[1], p, 1) == ERR_INVALID, family
                assert 'unknown tensor' in _error(), family
                assert _debug(L, family, h, dbg[0], p, 1) == ERR_STATE, family
                assert 'not written' in _error(), family
            for k, v in params:
                assert put(k, v) == capi.DFM_OK, (family, k, _error())
            assert count(h) == 0, family
            assert put(key, t) == capi.DFM_OK, family
            assert count(h) == 0, family
        finally:
            assert getattr(L, f'dfm_{family}_destroy')(h) == capi.DFM_OK
    assert seen == set(FAMILIES)
    for family in FAMILIES + ('box_post',):
        assert getattr(L, f'dfm_{family}_destroy')(None) == capi.DFM_OK, family
    assert L.dfm_neck_missing_params(None) == -1


def _unparameterised(L):
    """(family, handle at a small valid size, (a tensor a forward writes, an unknown name)) of
    the handles without parameters."""
    f8 = ctypes.c_float * 8
    ci8 = ctypes.c_int * 8
    anchors = (ctypes.c_float * (4 * 4 * 2 * 7))()   # ny = nx = 4, 2 anchors per cell
    half = f8(*[0.5] * 8)
    al = capi.AnchorLossDesc(1, 1, 2, 4, 4, 1, 0, 1, 1, 0, 0, f8(*[0.6] * 8), f8(*[0.45] * 8),
                             half, -1.0, 2.0, 0.25, 1.0 / 9, (ctypes.c_float * 4)(1, 2, 0.2, 0),
                             -1.5707963, 0.0, 0.0)
    at = capi.AtssLossDesc(1, 1, ci8(8), ci8(4), ci8(4), 1, 9, 8.0,
                           (ctypes.c_float * 4)(0.1, 0.1, 0.2, 0.2), 0.016, 1e-7, 2.0, 0.25,
                           (ctypes.c_float * 3)(1, 1, 1))
    ci2, cf2 = ctypes.c_int * 2, ctypes.c_float * 2
    ke = capi.KittiEvalDesc(1, (ctypes.c_int * 3)(0), 1, (ctypes.c_int * 3)(0), 0, 0,
                            (ctypes.c_double * 18)(*[0.7] * 18))
    return [
        ('anchor_loss', _create(L, 'anchor_loss', ctypes.byref(al), anchors), ('labels', 'nope')),
        ('atss_loss', _create(L, 'atss_loss', ctypes.byref(at)), ('labels', 'nope')),
        ('depth_loss', _create(L, 'depth_loss', ctypes.byref(capi.DepthLossDesc(
            1, 4, 4, 4, 1, 0, 2.0, 59.6, 1.0, 0.0, 1.0, 1.0, 0, 1.0))), ('count', 'nope')),
        ('imitation_loss', _create(L, 'imitation_loss', ctypes.byref(capi.ImitationLossDesc(
            1, 4, 4, 1, ci2(64), ci2(1), cf2(1.0), 10.0))), ('counts', 'nope')),
        ('box_post', _create(L, 'box_post', ctypes.byref(capi.BoxPostDesc(
            1, 2, 4, 4, 1, 1, -1, 10, 0.1, 0.01, -1.5707963, 0.0)), anchors),
         ('cls0_keep', 'cls1_keep')),
        ('kitti_eval', _create(L, 'kitti_eval', ctypes.byref(ke)), ('tp_scores', 'nope')),
    ]


@pytest.mark.gpu
def test_unparameterised_debug_hooks():
    """The handles without parameters keep the debug-hook part of the contract: an unknown name
    is DFM_ERR_INVALID before any forward too, a known one DFM_ERR_STATE until a forward ran;
    destroy(NULL) returns DFM_OK."""
    import torch
    L = capi.lib()
    buf = torch.zeros(1 << 16, device='cuda')
    p = vp(buf.data_ptr())
    for family, h, (known, unknown) in _unparameterised(L):
        try:
            assert _debug(L, family, h, unknown, p, 1) == ERR_INVALID, family
            assert 'unknown tensor' in _error(), (family, _error())
            assert _debug(L, family, h, known, p, 1) == ERR_STATE, family
            assert 'not written' in _error(), (family, _error())
        finally:
            assert getattr(L, f'dfm_{family}_destroy')(h) == capi.DFM_OK, family
        assert getattr(L, f'dfm_{family}_destroy')(None) == capi.DFM_OK, family


@pytest.mark.gpu
def test_debug_hook_checks_the_size_a_forward_wrote():
    """After a forward, a hook copies exactly what that forward wrote and refuses any other
    size (BEVHourglass's conv1: [Ny/2][Nx/2][128])."""
    import torch
    L = capi.lib()
    mirror = modules.BEVHourglass(64, 64, norm_cfg=GN)
    h = _create(L, 'bev_hourglass', ctypes.byref(capi.BevDesc(64, 64, 8, 8, 0)))
    try:
        for k, v in _uploaded(mirror):
            capi.check(L.dfm_bev_hourglass_set_param(h, k.encode(), vp(v.data_ptr()),
                                                     v.numel()), k)
        x = torch.zeros((64, 8, 8), device='cuda')
        out = torch.empty_like(x)
        capi.check(L.dfm_bev_hourglass_forward(h, vp(x.data_ptr()), None, vp(out.data_ptr()),
                                               None), 'dfm_bev_hourglass_forward')
        dst = torch.empty(4 * 4 * 128 + 1, device='cuda')
        d = vp(dst.data_ptr())
        assert _debug(L, 'bev_hourglass', h, 'conv1', d, 4 * 4 * 128 + 1) == ERR_INVALID
        assert 'elements' in _error()
        assert _debug(L, 'bev_hourglass', h, 'conv1', d, 4 * 4 * 128) == capi.DFM_OK
        torch.cuda.synchronize()
    finally:
        assert L.dfm_bev_hourglass_destroy(h) == capi.DFM_OK
