"""Host-side mirror of the reference's plugin interface for the DfM hot path.

Same class names, constructor arguments, ``state_dict`` keys, injected attributes
and return values as the reference modules, but ``forward`` hands raw device
pointers to the C-ABI library (``include/dfm_b200.h``) instead of running chains
of PyTorch ops:

    DfMBackbone          mmdet3d/models/backbones/dfm_backbone.py:14-214
    DepthHead            mmdet3d/models/dense_heads/depth_head.py:13-212
    DfMNeck              mmdet3d/models/necks/dfm_neck.py:10-122
    OutdoorImVoxelNeck   mmdet3d/models/necks/imvoxel_neck.py:8-68
    multiview_lift       mmdet3d/models/detectors/multiview_dfm.py:119-209
    FrustumToVoxel       mmdet3d/models/necks/feature_transformation.py:12-173
    Anchor3DHead         mmdet3d/models/dense_heads/anchor3d_head.py:139-185 (forward)
    SPPUNetNeck          mmdet3d/models/necks/spp_unet_neck.py (shipped KITTI config)
    FPN                  mmdet's FPN as the Waymo configs' image neck (mmdet 2.24 semantics)
    LIGAResNet           mmdet3d/models/backbones/liga_resnet.py (shipped KITTI config)

The ``nn.Conv3d`` / ``nn.GroupNorm`` / ``nn.BatchNorm3d`` children below are
parameter containers only (they give the exact reference ``state_dict`` layout so
reference checkpoints load with ``strict=True``); their ``forward`` is never
called.  There is no PyTorch fallback: without the built library or an H100 the
modules raise.
"""
import ctypes
import os

import numpy as np
import torch
import torch.nn as nn

from . import capi
from .registry import BACKBONES, HEADS, NECKS

_IMPL = {'auto': capi.DFM_CONV_AUTO, 'simt': capi.DFM_CONV_SIMT,
         'tc': capi.DFM_CONV_TC, 'tc_neck': capi.DFM_CONV_TC_NECK,
         'tc_neck_dhw': capi.DFM_CONV_TC_NECK_DHW}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_cuda(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError(
            f'{name} must be a CUDA tensor: depth_from_motion_b200 has no CPU path')
    if t.dtype != torch.float32:
        raise RuntimeError(f'{name} must be float32, got {t.dtype}')


_STRICT_PARAM_CHECK = bool(int(os.environ.get('DFM_PARAM_CHECK', '0')))


class _ParamSync:
    """Uploads parameters to a C handle whenever any of them changed.

    Change detection per forward is (storage pointer, tensor version) of every
    ``state_dict`` entry -- free, and it sees optimizer steps, ``copy_`` / ``fill_`` on
    the parameter, re-assignment and ``load_state_dict``.  It does NOT see in-place
    writes through ``param.data`` (``p.data.copy_(w)`` leaves ``p._version``
    untouched; EMA hooks and legacy init code do this).  Three safety nets:
    ``load_state_dict`` and ``train()`` / ``eval()`` always force a re-upload (the
    mirrors call ``mark_dirty`` from those hooks), callers that write through
    ``.data`` call ``module.sync_params()`` (or ``mark_dirty()``), and
    ``DFM_PARAM_CHECK=1`` adds a content fingerprint (sum and abs-sum of every
    tensor, one device sync per forward) for debugging such code."""

    def __init__(self):
        self._sig = None
        self._finger = None

    def mark_dirty(self):
        self._sig = None

    def signature(self, module):
        return tuple((k, v.data_ptr(), v._version)
                     for k, v in module.state_dict(keep_vars=True).items())

    @staticmethod
    def fingerprint(module):
        vals = [v.detach().double() for v in module.state_dict().values()
                if v.is_floating_point()]
        return torch.stack([torch.stack((v.sum(), v.abs().sum())) for v in vals]).cpu()

    def sync(self, module, set_fn):
        sig = self.signature(module)
        finger = self.fingerprint(module) if _STRICT_PARAM_CHECK else None
        if sig == self._sig and (finger is None or (
                self._finger is not None and torch.equal(finger, self._finger))):
            return
        for k, v in module.state_dict().items():
            if k.endswith('num_batches_tracked'):
                continue
            h = v.detach().to('cpu', torch.float32).contiguous()
            set_fn(k.encode(), ctypes.c_void_p(h.data_ptr()), h.numel())
        self._sig = sig
        self._finger = finger


class _CudaMirror(nn.Module):
    """Shared plumbing of the mirror modules: parameter re-upload hooks and the
    forward-only guard (the CUDA path has no backward; the reference trains these
    modules with autograd, which stays out of scope -- SURVEY.md section 3.3)."""

    def mark_dirty(self):
        """Force a parameter re-upload at the next forward (call after writing
        weights through ``param.data``)."""
        sync = getattr(self, '_sync', None)
        if sync is not None:
            sync.mark_dirty()

    sync_params = mark_dirty

    def train(self, mode=True):
        self.mark_dirty()
        return super().train(mode)

    def _load_from_state_dict(self, *args, **kwargs):
        self.mark_dirty()
        return super()._load_from_state_dict(*args, **kwargs)

    def _forward_only(self, *tensors):
        # eval-mode calls outside no_grad() just return tensors without a graph, which is
        # what inference code expects; training-mode calls would silently train nothing
        if not (self.training and torch.is_grad_enabled()):
            return
        if any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors) or \
                any(p.requires_grad for p in self.parameters()):
            raise RuntimeError(
                f'{type(self).__name__} (depth_from_motion_b200) is forward-only: call '
                '.eval() or run it under torch.no_grad(); autograd through the CUDA path '
                'is not implemented')


class _ConvGN(nn.Module):
    """Parameter layout of mmcv ConvModule(Conv3d, norm=GN): .conv / .gn."""

    def __init__(self, cin, cout, groups):
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, 3, 1, 1, bias=False)
        self.gn = nn.GroupNorm(groups, cout)


def _convbn3d(cin, cout, stride, groups):
    return nn.Sequential(nn.Conv3d(cin, cout, 3, stride, 1, bias=False),
                         nn.GroupNorm(groups, cout))


class _Hourglass(nn.Module):
    """Parameter layout of models/utils/conv_modules.py:73-127 (gn=True)."""

    def __init__(self, c):
        super().__init__()
        self.conv1 = nn.Sequential(_convbn3d(c, 2 * c, 2, 32), nn.ReLU(True))
        self.conv2 = _convbn3d(2 * c, 2 * c, 1, 32)
        self.conv3 = nn.Sequential(_convbn3d(2 * c, 2 * c, 2, 32), nn.ReLU(True))
        self.conv4 = nn.Sequential(_convbn3d(2 * c, 2 * c, 1, 32), nn.ReLU(True))
        self.conv5 = nn.Sequential(
            nn.ConvTranspose3d(2 * c, 2 * c, 3, padding=1, output_padding=1,
                               stride=2, bias=False), nn.GroupNorm(32, 2 * c))
        self.conv6 = nn.Sequential(
            nn.ConvTranspose3d(2 * c, c, 3, padding=1, output_padding=1,
                               stride=2, bias=False), nn.GroupNorm(32, c))


def geometry_from_meta(img_meta):
    """img_meta -> dfm_geometry_t (the fields dfm_backbone.py:150-172 reads)."""
    g = capi.Geometry()
    cam = np.asarray(img_meta['ori_cam2img'], dtype=np.float64)
    if cam.shape != (4, 4):
        pad = np.eye(4)
        pad[:cam.shape[0], :cam.shape[1]] = cam
        cam = pad
    c2p = img_meta['cur2prevs']
    if isinstance(c2p, torch.Tensor):
        c2p = c2p.detach().cpu().numpy()
    c2p = np.asarray(c2p, dtype=np.float64).reshape(-1, 4, 4)[0]
    g.cam2img[:] = cam.reshape(-1).tolist()
    g.cur2prev[:] = c2p.reshape(-1).tolist()
    crop = img_meta['crop_offset']
    g.crop_x, g.crop_y = float(crop[0]), float(crop[1])
    sf = img_meta.get('scale_factor', [1.0])
    g.scale = float(sf[0]) if hasattr(sf, '__len__') else float(sf)
    g.org_w = float(img_meta['ori_shape'][1])
    g.flip = int(bool(img_meta.get('flip', False)))
    return g


@BACKBONES.register_module()
class DfMBackbone(_CudaMirror):
    """Drop-in for the reference ``DfMBackbone`` (dfm_backbone.py:14-214)."""

    def __init__(self, in_channels, num_hg=1, cost_sample_factor=4,
                 feat_sample_factor=1, cv_channels=32,
                 depth_cfg=dict(mode='UD', num_bins=288, depth_min=2,
                                depth_max=59.6, downsample_factor=4),
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                 conv_impl='auto'):
        super().__init__()
        assert num_hg == 1, 'Only support num_hg=1 for now.'  # dfm_backbone.py:212
        assert norm_cfg.get('type') == 'GN', 'the reference hard-codes GN (:37)'
        self.norm_cfg = norm_cfg
        self.GN = True
        self.cost_sample_factor = cost_sample_factor
        self.feat_sample_factor = feat_sample_factor
        self.num_hg = num_hg
        self.cv_channels = cv_channels
        self.in_channels = in_channels
        self.depth_cfg = depth_cfg
        self.conv_impl = conv_impl
        groups = norm_cfg.get('num_groups', 32)
        # the kernels take GroupNorm statistics per group of C/32 channels
        # (nn.GroupNorm(32, C), conv_modules.py:42-43, which hard-codes 32 as well)
        assert groups == 32, 'only GroupNorm(num_groups=32) is implemented'
        cv = cv_channels

        def pred():
            return nn.Sequential(_ConvGN(cv, cv, groups),
                                 nn.Conv3d(cv, 1, 3, 1, 1, bias=False))

        self.dres0 = _ConvGN(2 * in_channels, cv, groups)
        self.dres1 = _ConvGN(cv, cv, groups)
        self.hg_stereo = nn.ModuleList([_Hourglass(cv)])
        self.pred_stereo = nn.ModuleList([pred()])
        self.dres0_mono = _ConvGN(in_channels, cv, groups)
        self.dres1_mono = _ConvGN(cv, cv, groups)
        self.hg_mono = nn.ModuleList([_Hourglass(cv)])
        self.pred_mono = nn.ModuleList([pred()])
        self.num_planes = round(depth_cfg['num_bins'] //
                                depth_cfg['downsample_factor'])
        self.aggregate_cost = nn.Conv2d(2 * self.num_planes, self.num_planes, 1,
                                        bias=False)
        self._handle = None
        self._handle_key = None
        self._sync = _ParamSync()
        self._depth_sig = None

    def init_weights(self):
        pass

    # ------------------------------------------------------------------
    def _default_depths(self):
        """DfM.prepare_depth (detectors/dfm.py:160-168), used when the detector has
        not injected ``downsampled_depth``."""
        cfg = self.depth_cfg
        ds = cfg['downsample_factor']
        interval = (cfg['depth_max'] - cfg['depth_min']) / cfg['num_bins']
        d = torch.zeros(cfg['num_bins'] // ds, dtype=torch.float32)
        for i in range(cfg['num_bins'] // ds):
            d[i] = (i + 0.5) * ds * interval + cfg['depth_min']
        return d

    def _ensure_handle(self, h, w):
        L = capi.lib()
        key = (h, w, self.conv_impl)
        if self._handle is not None and self._handle_key == key:
            return L
        self.release()
        desc = capi.BackboneDesc(self.in_channels, self.cv_channels, h, w,
                                 self.num_planes, self.cost_sample_factor,
                                 int(self.feat_sample_factor),
                                 _IMPL[self.conv_impl])
        hd = ctypes.c_void_p()
        capi.check(L.dfm_backbone_create(ctypes.byref(desc), ctypes.byref(hd)),
                   'dfm_backbone_create')
        self._handle, self._handle_key = hd, key
        self._sync = _ParamSync()
        self._depth_sig = None
        return L

    def release(self):
        if self._handle is not None:
            capi.lib().dfm_backbone_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def _prepare(self, h, w):
        L = self._ensure_handle(h, w)
        self._sync.sync(
            self, lambda k, p, n: capi.check(
                L.dfm_backbone_set_param(self._handle, k, p, n),
                f'dfm_backbone_set_param({k.decode()})'))
        depths = getattr(self, 'downsampled_depth', None)
        if depths is None:
            depths = self._default_depths()
        depths = depths.detach().to('cpu', torch.float32).contiguous()
        sig = depths.numpy().tobytes()
        if sig != self._depth_sig:
            capi.check(L.dfm_backbone_set_depths(
                self._handle, ctypes.c_void_p(depths.data_ptr()),
                depths.numel()), 'dfm_backbone_set_depths')
            self._depth_sig = sig
        return L

    def forward(self, cur_stereo_feats, prev_stereo_feats, img_metas,
                cur_sem_feats=None):
        _check_cuda(cur_stereo_feats, 'cur_stereo_feats')
        _check_cuda(prev_stereo_feats, 'prev_stereo_feats')
        self._forward_only(cur_stereo_feats, prev_stereo_feats)
        b, c, h, w = cur_stereo_feats.shape
        # the reference only supports batch size 1 (dfm_backbone.py:160, SURVEY 8a)
        assert b == 1, 'only support batch size 1 for now'
        assert c == self.in_channels
        assert prev_stereo_feats.shape == cur_stereo_feats.shape
        L = self._prepare(h, w)
        cur = cur_stereo_feats.contiguous()
        prev = prev_stereo_feats.contiguous()
        geom = geometry_from_meta(img_metas[0])
        ho = round(h / self.cost_sample_factor)
        wo = round(w / self.cost_sample_factor)
        d = self.num_planes
        dev = cur.device
        cost = torch.empty((1, 1, d, ho, wo), device=dev, dtype=torch.float32)
        stereo = torch.empty((1, self.cv_channels, d, ho, wo), device=dev,
                             dtype=torch.float32)
        mono = torch.empty_like(stereo)
        # stereo features that came out of our SPPUNetNeckTail carry a channels-last twin:
        # the plane-sweep loader reads it directly, no NCHW -> NHWC transposes
        cl_c = getattr(cur_stereo_feats, '_dfm_cl', None)
        cl_p = getattr(prev_stereo_feats, '_dfm_cl', None)
        if cl_c is not None and cl_p is not None and cl_c.shape == (h, w, c) == cl_p.shape:
            capi.check(L.dfm_backbone_forward_cl(
                self._handle, _ptr(cl_c), _ptr(cl_p), ctypes.byref(geom), _ptr(cost),
                _ptr(stereo), _ptr(mono), _stream()), 'dfm_backbone_forward_cl')
        else:
            capi.check(L.dfm_backbone_forward(
                self._handle, _ptr(cur), _ptr(prev), ctypes.byref(geom), _ptr(cost),
                _ptr(stereo), _ptr(mono), _stream()), 'dfm_backbone_forward')
        # the handle keeps a channels-last copy of stereo_feat until the next forward;
        # FrustumToVoxel reads it instead of transposing `stereo` again
        self._generation = getattr(self, '_generation', 0) + 1
        stereo._dfm_channels_last = (self, self._generation)
        return cost, stereo, mono

    def debug_tensor(self, name, shape):
        """Channels-last copy of an intermediate (tests only)."""
        return _debug_tensor(self._handle, 'dfm_backbone_debug_tensor', name, shape)


def _debug_tensor(handle, fn, name, shape):
    """Channels-last copy of the intermediate `name` the handle's last forward wrote, through
    the test hook `fn` of include/dfm_b200.h (shape must hold exactly that tensor)."""
    if handle is None:
        raise RuntimeError(f'{fn}: no forward has run')
    out = torch.empty(shape, device='cuda', dtype=torch.float32)
    capi.check(getattr(capi.lib(), fn)(handle, name.encode(), _ptr(out), out.numel(), _stream()),
               f'{fn}({name})')
    return out


def build_dfm_cost(cur_feats, prev_feats, depths, feat_sample_factor,
                   cost_sample_factor, cam2imgs, cur2prevs, img_shape,
                   flip=False, img_crop_offset=(0, 0), img_scale_factor=1.0):
    """Same signature as dfm_backbone.py:217-227; materialises the
    [1, 2C, D, Ho, Wo] volume with the CUDA warp kernel (parity op)."""
    _check_cuda(cur_feats, 'cur_feats')
    b, c, h, w = cur_feats.shape
    assert b == 1
    meta = dict(ori_cam2img=torch.as_tensor(cam2imgs)[0].cpu().numpy(),
                cur2prevs=torch.as_tensor(cur2prevs).cpu().numpy(),
                crop_offset=img_crop_offset, scale_factor=[img_scale_factor],
                ori_shape=(img_shape[0], img_shape[1], 3), flip=flip)
    geom = geometry_from_meta(meta)
    depths = depths.detach().to('cpu', torch.float32).contiguous()
    d = depths.numel()
    ho, wo = round(h / cost_sample_factor), round(w / cost_sample_factor)
    out = torch.empty((1, 2 * c, d, ho, wo), device=cur_feats.device,
                      dtype=torch.float32)
    capi.check(capi.lib().dfm_op_build_cost_volume(
        _ptr(cur_feats.contiguous()), _ptr(prev_feats.contiguous()), c, h, w,
        ctypes.c_void_p(depths.data_ptr()), d, cost_sample_factor,
        int(feat_sample_factor), ctypes.byref(geom), _ptr(out), _stream()),
        'dfm_op_build_cost_volume')
    return out


def conv3d(x, weight, stride=(1, 1, 1), padding=(1, 1, 1), transposed=False,
           impl='auto'):
    """3x3x3 conv3d / conv_transpose3d(k3,s2,p1,op1) building block (NCDHW)."""
    _check_cuda(x, 'x')
    n, cin, di, hi, wi = x.shape
    assert n == 1
    cout = weight.shape[1] if transposed else weight.shape[0]
    if transposed:
        do, ho, wo = 2 * di, 2 * hi, 2 * wi
    else:
        do = (di + 2 * padding[0] - 3) // stride[0] + 1
        ho = (hi + 2 * padding[1] - 3) // stride[1] + 1
        wo = (wi + 2 * padding[2] - 3) // stride[2] + 1
    y = torch.empty((1, cout, do, ho, wo), device=x.device, dtype=torch.float32)
    wh = weight.detach().to('cpu', torch.float32).contiguous()
    st = (ctypes.c_int * 3)(*stride)
    pd = (ctypes.c_int * 3)(*padding)
    capi.check(capi.lib().dfm_op_conv3d(
        _ptr(x.contiguous()), cin, di, hi, wi, ctypes.c_void_p(wh.data_ptr()),
        cout, st, pd, int(transposed), _IMPL[impl], _ptr(y), _stream()),
        'dfm_op_conv3d')
    return y


@HEADS.register_module()
class DepthHead(_CudaMirror):
    """Drop-in for the reference ``DepthHead`` forward (depth_head.py:13-212).
    ``loss`` is training-side PyTorch in the reference and is out of scope
    (SURVEY.md section 8a row a5)."""

    def __init__(self, depth_cfg, in_channels=32, with_convs=True,
                 depth_loss=dict(type='ce', loss_weight=1.0),
                 downsample_factor=4, num_views=5,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)):
        super().__init__()
        self.in_channels = in_channels
        self.depth_cfg = depth_cfg
        self.with_convs = with_convs
        self.depth_loss = depth_loss
        self.downsample_factor = downsample_factor
        self.num_views = num_views
        self.norm_cfg = norm_cfg
        self.depth_loss_type = depth_loss['type']
        self.loss_weight = depth_loss['loss_weight']
        self.min_depth = depth_cfg['min_depth']
        self.max_depth = depth_cfg['max_depth']
        if self.with_convs:
            self.conv_depth = nn.Conv3d(in_channels, 1, 3, 1, 1, bias=False)
        self._samples_dev = None

    def forward(self, stereo_features, return_volumes=True):
        """Returns (depth_volumes, depth_volumes_softmax, depth_preds) like
        depth_head.py:190-212.  ``return_volumes=False`` skips the two
        [B,N,fD,fH,fW] outputs (returns None for them)."""
        _check_cuda(stereo_features, 'stereo_features')
        self._forward_only(stereo_features)
        if self.with_convs:
            raise NotImplementedError(
                'DepthHead(with_convs=True) is not on the shipped DfM path '
                '(configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:126 uses False)')
        b, n, d, h, w = stereo_features.shape
        f = self.downsample_factor
        samples = self.depth_samples
        if (self._samples_dev is None or self._samples_dev[0] is not samples
                or self._samples_dev[1].device != stereo_features.device):
            self._samples_dev = (samples, samples.detach().to(
                stereo_features.device, torch.float32).contiguous())
        sdev = self._samples_dev[1]
        assert sdev.numel() == f * d
        x = stereo_features.contiguous()
        dev = x.device
        vol = sm = None
        if return_volumes:
            vol = torch.empty((b, n, f * d, f * h, f * w), device=dev)
            sm = torch.empty_like(vol)
        preds = torch.empty((b, n, f * h, f * w), device=dev)
        L = capi.lib()
        for i in range(b * n):
            bi, ni = divmod(i, n)
            capi.check(L.dfm_depth_head_forward(
                _ptr(x[bi, ni]), _ptr(sdev), d, h, w, f,
                _ptr(vol[bi, ni]) if vol is not None else None,
                _ptr(sm[bi, ni]) if sm is not None else None,
                _ptr(preds[bi, ni]), _stream()), 'dfm_depth_head_forward')
        return vol, sm, preds


class _NeckBase(_CudaMirror):
    def _make_tower(self, c0, c1, c2, cout):
        def cm(ci, co, **kw):
            m = nn.Module()
            m.conv = nn.Conv3d(ci, co, 3, bias=False, **kw)
            m.bn = nn.BatchNorm3d(co)
            return m

        def res(c):
            m = nn.Module()
            m.conv0 = cm(c, c, padding=1)
            m.conv1 = cm(c, c, padding=1)
            return m

        return nn.Sequential(res(c0), cm(c0, c1, stride=(1, 1, 2), padding=1),
                             res(c1), cm(c1, c2, stride=(1, 1, 2), padding=1),
                             res(c2), cm(c2, cout, padding=(1, 1, 0)))

    def _run(self, x, num_frames, conv_impl):
        _check_cuda(x, 'x')
        assert not self.training, \
            'the CUDA necks fold BatchNorm3d running statistics: call .eval()'
        n, c, nx, ny, nz = x.shape
        L = capi.lib()
        key = (nx, ny, nz, conv_impl)
        if getattr(self, '_handle', None) is None or self._handle_key != key:
            self.release()
            desc = capi.NeckDesc(self._c0, self._cout, num_frames, nx, ny, nz,
                                 _IMPL[conv_impl])
            hd = ctypes.c_void_p()
            capi.check(L.dfm_neck_create(ctypes.byref(desc), ctypes.byref(hd)),
                       'dfm_neck_create')
            self._handle, self._handle_key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_neck_set_param(self._handle, k, p, m),
            f'dfm_neck_set_param({k.decode()})'))
        outs = []
        for i in range(n):
            bev = torch.empty((self._cout, ny, nx), device=x.device)
            xi = x[i]
            if xi.permute(1, 2, 3, 0).is_contiguous():   # channels-last (multiview_lift's output)
                capi.check(L.dfm_neck_forward_cl(self._handle, _ptr(xi), _ptr(bev), _stream()),
                           'dfm_neck_forward_cl')
            else:
                capi.check(L.dfm_neck_forward(self._handle, _ptr(xi.contiguous()),
                                              _ptr(bev), _stream()),
                           'dfm_neck_forward')
            outs.append(bev)
        return [torch.stack(outs)]

    def debug_tensor(self, name, shape):
        """Raw output of conv layer i of a tower, [Nx, Ny, Zo, C] ('mono.<i>' / 'stereo.<i>';
        OutdoorImVoxelNeck's one tower is 'mono'), from the last forward (tests only)."""
        return _debug_tensor(getattr(self, '_handle', None), 'dfm_neck_debug_tensor', name, shape)

    def release(self):
        if getattr(self, '_handle', None) is not None:
            capi.lib().dfm_neck_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def init_weights(self):
        pass


@NECKS.register_module()
class OutdoorImVoxelNeck(_NeckBase):
    """Drop-in for imvoxel_neck.py:8-68 (eval mode)."""

    def __init__(self, in_channels, out_channels, norm_cfg=dict(type='BN3d'),
                 output_bev=True, conv_impl='auto'):
        super().__init__()
        assert norm_cfg.get('type') == 'BN3d' and output_bev
        self.output_bev = output_bev
        if not isinstance(in_channels, list):
            in_channels = [in_channels, in_channels * 2, in_channels * 4]
        self.in_channels = in_channels
        self._c0, self._cout = in_channels[0], out_channels
        assert in_channels[1] == 2 * in_channels[0]
        assert in_channels[2] == 4 * in_channels[0]
        self.conv_impl = conv_impl
        self.model = self._make_tower(*in_channels, out_channels)
        self._handle = None

    def forward(self, x):
        return self._run(x, 0, self.conv_impl)


@NECKS.register_module()
class DfMNeck(_NeckBase):
    """Drop-in for dfm_neck.py:10-122 (eval mode)."""

    def __init__(self, in_channels, out_channels, norm_cfg=dict(type='BN3d'),
                 num_frames=2, conv_impl='auto'):
        super().__init__()
        assert norm_cfg.get('type') == 'BN3d'
        if not isinstance(in_channels, list):
            in_channels = [in_channels, in_channels * 2, in_channels * 4]
        self.in_channels = in_channels
        self.num_frames = num_frames
        self._c0, self._cout = in_channels[0], out_channels
        self.conv_impl = conv_impl
        self.mono_layers = self._make_tower(*in_channels, out_channels)
        self.stereo_layers = self._make_tower(in_channels[0] * num_frames,
                                              in_channels[1], in_channels[2],
                                              out_channels)
        self.aggregate_layer = nn.Conv2d(2 * out_channels, 1, 1, bias=False)
        self._handle = None

    def forward(self, x):
        assert x.shape[1] == self.in_channels[0] * self.num_frames
        return self._run(x, self.num_frames, self.conv_impl)


class CostLogits:
    """Marks a ``[B, 1, D, H, W]`` tensor of low-res cost logits (DfMBackbone's
    first output) handed to ``FrustumToVoxel.forward`` in place of
    ``stereo_feat_softmax``: the depth distribution is then evaluated from the
    logits inside the sampling kernel and the x4-upsampled ``[B, 1, 4D, 4H, 4W]``
    softmax volume (depth_head.py:196-204) is never materialised.  With
    ``depth_samples`` (the tensor the detector injects into DepthHead,
    detectors/dfm.py:90) the same pass also produces DepthHead's ``depth_preds``,
    left in ``self.depth_preds`` after the call."""

    def __init__(self, cost, depth_samples=None):
        self.cost = cost
        self.depth_samples = depth_samples
        self.depth_preds = None


@NECKS.register_module()
class FrustumToVoxel(_CudaMirror):
    """Drop-in for the reference ``FrustumToVoxel``
    (necks/feature_transformation.py:12-173): same constructor arguments and
    ``state_dict`` keys (``voxel_convs.<i>.0.conv.weight`` /
    ``voxel_convs.<i>.0.gn.{weight,bias}``); ``depth_cfg`` and ``coordinates_3d``
    are injected by the detector exactly like the reference
    (detectors/dfm.py:85-100)."""

    def __init__(self, num_3dconvs=1, cv_channels=32, out_channels=32,
                 in_sem_channels=32, sem_atten_feat=True,
                 stereo_atten_feat=False, cat_img_feature=True,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                 conv_impl='auto'):
        super().__init__()
        self.GN = True
        self.num_3dconvs = num_3dconvs
        self.cv_channels = cv_channels
        self.out_channels = out_channels
        self.in_sem_channels = in_sem_channels
        self.sem_atten_feat = sem_atten_feat
        self.stereo_atten_feat = stereo_atten_feat
        self.cat_img_feature = bool(cat_img_feature)
        self.conv_impl = conv_impl
        assert norm_cfg['type'] == 'GN' and norm_cfg['num_groups'] == 32
        cin = cv_channels + (in_sem_channels if self.cat_img_feature else 0)
        self.voxel_convs = nn.Sequential(*[
            nn.Sequential(_ConvGN(cin if i == 0 else out_channels,
                                  out_channels, 32))
            for i in range(num_3dconvs)])
        self._handle = None
        self._key = None

    def init_weights(self):
        pass

    def debug_tensor(self, name, shape):
        """'vox' ([nz, ny, nx, cv], the gathered conv input) or 'conv<i>' (raw output of
        voxel_convs[i], [nz, ny, nx, 32]) of the last forward (tests only)."""
        return _debug_tensor(self._handle, 'dfm_frustum_debug_tensor', name, shape)

    def release(self):
        if getattr(self, '_handle', None) is not None:
            capi.lib().dfm_frustum_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    @staticmethod
    def _separable_centres(c3d):
        """coordinates_3d is a meshgrid of three linspaces (detectors/dfm.py:
        193-211); the kernel takes the three axes."""
        c3d = c3d.detach().to('cpu', torch.float32)
        xs = c3d[0, 0, :, 0].contiguous()
        ys = c3d[0, :, 0, 1].contiguous()
        zs = c3d[:, 0, 0, 2].contiguous()
        ok = (torch.equal(c3d[..., 0], xs[None, None, :].expand(c3d.shape[:3]))
              and torch.equal(c3d[..., 1], ys[None, :, None].expand(c3d.shape[:3]))
              and torch.equal(c3d[..., 2], zs[:, None, None].expand(c3d.shape[:3])))
        if not ok:
            raise RuntimeError('coordinates_3d is not a separable (meshgrid) voxel grid')
        return xs, ys, zs

    def _ensure_handle(self, d, h, w, sh, sw, f):
        c3d = self.coordinates_3d
        key = (d, h, w, sh, sw, f, tuple(c3d.shape), c3d.data_ptr(),
               c3d._version, float(self.depth_cfg['depth_min']),
               float(self.depth_cfg['depth_max']))
        if self._handle is not None and key == self._key:
            return
        self.release()
        xs, ys, zs = self._separable_centres(c3d)
        nz, ny, nx = c3d.shape[:3]
        desc = capi.FrustumDesc(
            self.num_3dconvs, self.cv_channels, self.out_channels,
            self.in_sem_channels, int(self.sem_atten_feat),
            int(self.stereo_atten_feat), int(self.cat_img_feature), d, h, w, sh,
            sw, f, nx, ny, nz, float(self.depth_cfg['depth_min']),
            float(self.depth_cfg['depth_max']), _IMPL[self.conv_impl])
        hd = ctypes.c_void_p()
        capi.check(capi.lib().dfm_frustum_create(
            ctypes.byref(desc), _ptr(xs), _ptr(ys), _ptr(zs), ctypes.byref(hd)),
            'dfm_frustum_create')
        self._handle, self._key = hd, key
        self._sync = _ParamSync()

    def forward(self, stereo_feat, stereo_feat_softmax, img_metas,
                cur_sem_feats=None):
        """feature_transformation.py:68-173.  ``stereo_feat_softmax`` is the
        DepthHead's ``[B, 1, fD, fH, fW]`` tensor like in the reference, or a
        ``CostLogits`` wrapper (fused path)."""
        _check_cuda(stereo_feat, 'stereo_feat')
        self._forward_only(stereo_feat, cur_sem_feats)
        b, c, d, h, w = stereo_feat.shape
        assert b == len(img_metas)
        logits = sm = samples = preds = None
        if isinstance(stereo_feat_softmax, CostLogits):
            logits = stereo_feat_softmax.cost.contiguous()
            _check_cuda(logits, 'cost logits')
            assert tuple(logits.shape) == (b, 1, d, h, w)
            f = int(self.depth_cfg.get('downsample_factor', 4))
            if stereo_feat_softmax.depth_samples is not None:
                samples = stereo_feat_softmax.depth_samples.detach().to(
                    logits.device, torch.float32).contiguous()
                assert samples.numel() == f * d
                preds = torch.empty((b, 1, f * h, f * w), device=logits.device)
                stereo_feat_softmax.depth_preds = preds
        elif stereo_feat_softmax is not None:
            sm = stereo_feat_softmax.contiguous()
            _check_cuda(sm, 'stereo_feat_softmax')
            f = sm.shape[2] // d
            assert tuple(sm.shape) == (b, 1, f * d, f * h, f * w)
        else:
            f = 1
        sem = None
        sh = sw = 1
        if self.cat_img_feature:
            _check_cuda(cur_sem_feats, 'cur_sem_feats')
            sem = cur_sem_feats.contiguous()
            sh, sw = sem.shape[-2:]
        self._ensure_handle(d, h, w, sh, sw, f)
        L = capi.lib()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_frustum_set_param(self._handle, k, p, m),
            f'dfm_frustum_set_param({k.decode()})'))
        nz, ny, nx = self.coordinates_3d.shape[:3]
        pad = img_metas[0]['pad_shape']
        x = stereo_feat.contiguous()
        out = torch.empty((b, self.out_channels, nz // 4, ny, nx),
                          device=x.device)
        # a stereo_feat that came straight out of our DfMBackbone has a live
        # channels-last twin inside the backbone handle: no transpose needed
        tag = getattr(stereo_feat, '_dfm_channels_last', None)
        twin = None
        if (tag is not None and b == 1 and tag[0]._handle is not None
                and tag[0]._generation == tag[1]):
            twin = L.dfm_backbone_stereo_feat_device(tag[0]._handle)
        for i in range(b):
            P = (ctypes.c_double * 16)(*np.asarray(
                img_metas[i]['cam2img'], np.float64).reshape(-1)[:16].tolist())
            capi.check(L.dfm_frustum_forward(
                self._handle,
                ctypes.c_void_p(twin) if twin else _ptr(x[i]),
                capi.DFM_LAYOUT_DHWC if twin else capi.DFM_LAYOUT_NCDHW,
                _ptr(sm[i]) if sm is not None else None,
                _ptr(logits[i]) if logits is not None else None,
                _ptr(samples), _ptr(preds[i]) if preds is not None else None,
                _ptr(sem[i]) if sem is not None else None, P, int(pad[0]),
                int(pad[1]), _ptr(out[i]), _stream()), 'dfm_frustum_forward')
        return out


class HotPathPipeline:
    """``DfM.simple_test``'s hot-path segment as one C-ABI call with HOST buffers
    (detectors/dfm.py:296, :420, :423-425): ``backbone_stereo`` -> ``depth_head``
    -> ``feature_transformation``.  Pinned host features in, pinned host voxel
    features + ``depth_preds`` out; nothing else leaves the device.  This is the call
    a deployment that keeps the 2-D backbone and the BEV head in PyTorch makes once per
    frame (``bench.py``'s ``e2e`` number times it)."""

    def __init__(self, backbone, depth_head, frustum):
        self.backbone, self.depth_head, self.frustum = backbone, depth_head, frustum
        self._outs = None
        self._slot = 0
        self._inflight = []

    def prepare(self, feat_h, feat_w, sem_hw):
        bb, fr = self.backbone, self.frustum
        L = bb._prepare(feat_h, feat_w)
        ho = round(feat_h / bb.cost_sample_factor)
        wo = round(feat_w / bb.cost_sample_factor)
        f = int(self.depth_head.downsample_factor)
        fr._ensure_handle(bb.num_planes, ho, wo, sem_hw[0], sem_hw[1], f)
        fr._sync.sync(fr, lambda k, p, m: capi.check(
            L.dfm_frustum_set_param(fr._handle, k, p, m),
            f'dfm_frustum_set_param({k.decode()})'))
        nz, ny, nx = fr.coordinates_3d.shape[:3]
        if self._outs is None or self._outs[0][0].shape[-3:] != (nz // 4, ny, nx) or \
                self._outs[0][1].shape[-2:] != (f * ho, f * wo):
            # two pinned output sets: frame i's results are read while frame i+1 is in flight
            self._outs = [(torch.empty((1, fr.out_channels, nz // 4, ny, nx)).pin_memory(),
                           torch.empty((1, 1, f * ho, f * wo)).pin_memory()) for _ in range(2)]
            self._samples = self.depth_head.depth_samples.detach().to(
                'cpu', torch.float32).contiguous()
        return L

    @property
    def _out(self):
        return self._outs[0]

    def prefetch(self, h_cur, h_prev, h_sem=None):
        """Start copying the NEXT frame's inputs (pinned host tensors) while the current one
        runs.  Pass ``h_sem`` too: a host->device copy issued at submit time queues on the copy
        engine behind this bulk copy and stalls the compute stream."""
        if self.backbone._handle is None:
            self.backbone._prepare(h_cur.shape[-2], h_cur.shape[-1])
        capi.check(capi.lib().dfm_pipeline_prefetch_host(
            self.backbone._handle, _ptr(h_cur), _ptr(h_prev), _ptr(h_sem),
            0 if h_sem is None else h_sem.numel()), 'dfm_pipeline_prefetch_host')

    def _args(self, h_cur, h_prev, h_sem, img_metas):
        for t in (h_cur, h_prev):
            assert t.device.type == 'cpu' and t.dtype == torch.float32 and t.is_contiguous()
        _, _, h, w = h_cur.shape
        L = self.prepare(h, w, tuple(h_sem.shape[-2:]) if h_sem is not None else (1, 1))
        meta = img_metas[0]
        geom = geometry_from_meta(meta)
        P = (ctypes.c_double * 16)(*np.asarray(
            meta['cam2img'], np.float64).reshape(-1)[:16].tolist())
        pad = meta['pad_shape']
        return L, geom, P, int(pad[0]), int(pad[1])

    def __call__(self, h_cur, h_prev, h_sem, img_metas, h_cost=None):
        """Synchronous call.  h_cur / h_prev [1,C,H,W], h_sem [1,32,H/4,W/4]: CPU float32
        tensors (pinned for full PCIe bandwidth).  Returns (voxel_features [1,32,Nz/4,Ny,Nx],
        depth_preds [1,1,H,W]) as pinned CPU tensors owned by this object (overwritten by a
        later call)."""
        L, geom, P, ph, pw = self._args(h_cur, h_prev, h_sem, img_metas)
        self._inflight = []
        vox, preds = self._outs[self._slot]
        self._slot ^= 1
        capi.check(L.dfm_pipeline_forward_host(
            self.backbone._handle, self.frustum._handle, _ptr(h_cur), _ptr(h_prev),
            _ptr(h_sem), ctypes.byref(geom), P, ph, pw, _ptr(self._samples), _ptr(vox),
            _ptr(preds), _ptr(h_cost), _stream()), 'dfm_pipeline_forward_host')
        return vox, preds

    def submit(self, h_cur, h_prev, h_sem, img_metas):
        """Asynchronous call: enqueue one frame and return at once (at most two in flight).
        ``wait()`` returns the outputs of the oldest submitted frame; the device->host copy of
        frame i overlaps the compute of frame i+1."""
        L, geom, P, ph, pw = self._args(h_cur, h_prev, h_sem, img_metas)
        vox, preds = self._outs[self._slot]
        capi.check(L.dfm_pipeline_submit_host(
            self.backbone._handle, self.frustum._handle, _ptr(h_cur), _ptr(h_prev),
            _ptr(h_sem), ctypes.byref(geom), P, ph, pw, _ptr(self._samples), _ptr(vox),
            _ptr(preds), _stream()), 'dfm_pipeline_submit_host')
        self._slot ^= 1
        self._inflight.append((vox, preds, h_cur, h_prev, h_sem))

    def wait(self):
        capi.check(capi.lib().dfm_pipeline_wait(self.backbone._handle), 'dfm_pipeline_wait')
        vox, preds = self._inflight.pop(0)[:2]
        return vox, preds


class _ConvGN2d(nn.Module):
    """Parameter layout of mmcv ConvModule(Conv2d 3x3, norm=GN): .conv / .gn."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 3, 1, 1, bias=False)
        self.gn = nn.GroupNorm(32, cout)


def _convbn2d(cin, cout, stride):
    return nn.Sequential(nn.Conv2d(cin, cout, 3, stride, 1, bias=False),
                         nn.GroupNorm(32, cout))


class _Hourglass2d(nn.Module):
    """Parameter layout of hourglass2d (backbones/bev_hourglass.py:53-119, gn=True)."""

    def __init__(self, c):
        super().__init__()
        self.conv1 = nn.Sequential(_convbn2d(c, 2 * c, 2), nn.ReLU(True))
        self.conv2 = _convbn2d(2 * c, 2 * c, 1)
        self.conv3 = nn.Sequential(_convbn2d(2 * c, 2 * c, 2), nn.ReLU(True))
        self.conv4 = nn.Sequential(_convbn2d(2 * c, 2 * c, 1), nn.ReLU(True))
        self.conv5 = nn.Sequential(
            nn.ConvTranspose2d(2 * c, 2 * c, 3, padding=1, output_padding=1, stride=2,
                               bias=False), nn.GroupNorm(32, 2 * c))
        self.conv6 = nn.Sequential(
            nn.ConvTranspose2d(2 * c, c, 3, padding=1, output_padding=1, stride=2,
                               bias=False), nn.GroupNorm(32, c))


class _HandleMirror(_CudaMirror):
    """create / destroy / parameter-sync plumbing shared by the 2-D BEV mirrors."""
    _destroy = None

    def release(self):
        if getattr(self, '_handle', None) is not None:
            getattr(capi.lib(), self._destroy)(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def init_weights(self):
        pass


@NECKS.register_module()
class SPPUNetNeckTail(_HandleMirror):
    """The last two layers of the reference ``SPPUNetNeck`` (necks/spp_unet_neck.py:60-75
    ``lastconv``, applied at :110) on CUDA: 3x3 conv + GroupNorm(32) + ReLU + 1x1 conv on the
    full-resolution up-convolved feature.  ``state_dict`` keys are the reference's
    (``lastconv.0.conv.weight``, ``lastconv.0.gn.*``, ``lastconv.1.weight``), so
    ``load_state_dict(neck.state_dict(), strict=False)`` of a reference neck fills it.  The
    returned ``[B, 32, H, W]`` tensor carries a channels-last twin that our ``DfMBackbone``
    consumes directly.  Patch: ``neck.lastconv = SPPUNetNeckTail(...)`` (it is called with the
    same single tensor argument as the ``nn.Sequential`` it replaces)."""
    _destroy = 'dfm_stereo_tail_destroy'

    def __init__(self, stereo_channels=(32, 32), in_channels=32,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), conv_impl='auto'):
        super().__init__()
        assert tuple(stereo_channels) == (32, 32) and in_channels == 32
        assert norm_cfg.get('type') == 'GN' and norm_cfg.get('num_groups', 32) == 32
        self.conv_impl = conv_impl
        self.lastconv = nn.Sequential(_ConvGN2d(32, 32), nn.Conv2d(32, 32, 1, bias=False))
        self._handle = None
        self._key = None

    def forward(self, x):
        _check_cuda(x, 'x')
        self._forward_only(x)
        b, c, h, w = x.shape
        assert c == 32
        L = capi.lib()
        key = (h, w, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            hd = ctypes.c_void_p()
            capi.check(L.dfm_stereo_tail_create(h, w, _IMPL[self.conv_impl], ctypes.byref(hd)),
                       'dfm_stereo_tail_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_stereo_tail_set_param(self._handle, k, p, m),
            f'dfm_stereo_tail_set_param({k.decode()})'))
        x = x.contiguous()
        out = torch.empty_like(x)
        twins = []
        for i in range(b):
            cl = torch.empty((h, w, c), device=x.device)
            capi.check(L.dfm_stereo_tail_forward(self._handle, _ptr(x[i]), _ptr(cl),
                                                 _ptr(out[i]), _stream()),
                       'dfm_stereo_tail_forward')
            twins.append(cl)
        if b == 1:
            out._dfm_cl = twins[0]
        return out


class _ConvGN1x1(nn.Module):
    """Parameter layout of mmcv ConvModule(Conv2d 1x1, norm=GN): .conv / .gn."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1, bias=False)
        self.gn = nn.GroupNorm(32, cout)


def _convbn_bn(cin, cout):
    """Parameter layout of models/utils/conv_modules.py:6-24 ``convbn`` (SyncBatchNorm: the
    BatchNorm2d placeholder has the same state_dict, num_batches_tracked included)."""
    return nn.Sequential(nn.Conv2d(cin, cout, 3, 1, 1, bias=False), nn.BatchNorm2d(cout))


class _UpconvModule(nn.Module):
    """Parameter layout of models/utils/conv_modules.py:46-60 ``upconv_module([512, 64, 3],
    [64, 32])``."""

    def __init__(self):
        super().__init__()
        self.conv = nn.ModuleList([_convbn_bn(512, 64), _convbn_bn(64, 32)])
        self.redir = nn.ModuleList([_convbn_bn(64, 64), _convbn_bn(3, 32)])


@NECKS.register_module()
class SPPUNetNeck(_HandleMirror):
    """The reference ``SPPUNetNeck`` (necks/spp_unet_neck.py) of the shipped KITTI config on
    CUDA: SPP branches, concat, ``upconv_module``, ``lastconv`` and ``rpnconv``
    (``csrc/spp_neck_api.inc``).  ``forward(feats) -> (stereo_feature [B, 32, H, W],
    sem_feature [B, 32, H/4, W/4])`` for ``feats = [img, f1, f2, f3, f4]`` (NCHW, LIGAResNet34's
    [3 @ H, 64 @ H/2, 128 @ H/4 x 3]).  The ``state_dict`` is the reference's (46 entries, BN
    running statistics included); BatchNorm runs in eval form.  For B == 1 the stereo feature
    carries a channels-last twin that our ``DfMBackbone`` consumes without transposes.
    Patch: ``model.neck = SPPUNetNeck(**cfg.model.neck)``."""
    _destroy = 'dfm_spp_neck_destroy'

    def __init__(self, in_channels, start_level, sem_channels=[128, 32], stereo_channels=[32, 32],
                 spp_channel=32, with_upconv=True, cat_img_feature=True, norm_cfg=None,
                 conv_impl='auto'):
        super().__init__()
        assert list(in_channels) == [3, 64, 128, 128, 128] and start_level == 2, \
            'only the shipped KITTI configuration is implemented'
        assert list(sem_channels) == [128, 32] and list(stereo_channels) == [32, 32]
        assert spp_channel == 32 and with_upconv and cat_img_feature
        assert norm_cfg is not None and norm_cfg.get('type') == 'GN' and \
            norm_cfg.get('num_groups', 32) == 32, 'only the GroupNorm(32) variant is implemented'
        self.in_channels, self.start_level = list(in_channels), start_level
        self.sem_channels, self.stereo_channels = list(sem_channels), list(stereo_channels)
        self.spp_channel, self.with_upconv = spp_channel, with_upconv
        self.cat_img_feature = cat_img_feature
        self.conv_impl = conv_impl
        self.spp_branches = nn.ModuleList([
            nn.Sequential(nn.AvgPool2d(s, stride=s), _ConvGN1x1(128, 32))
            for s in (64, 32, 16, 8)])
        self.upconv_module = _UpconvModule()
        self.lastconv = nn.Sequential(_ConvGN2d(32, 32), nn.Conv2d(32, 32, 1, bias=False))
        self.rpnconv = nn.Sequential(_ConvGN2d(512, 128), _ConvGN2d(128, 32))
        self._handle = None
        self._key = None

    @staticmethod
    def check_shapes(feats):
        """Raises ValueError on the inputs the reference rejects (or cannot add up)."""
        if len(feats) != 5:
            raise ValueError(f'SPPUNetNeck takes 5 feature maps, got {len(feats)}')
        img, f1, f2, f3, f4 = feats
        b, _, h, w = img.shape
        want = ((b, 3, h, w), (b, 64, h // 2, w // 2)) + ((b, 128, h // 4, w // 4),) * 3
        got = tuple(tuple(f.shape) for f in feats)
        if h % 4 or w % 4 or got != want:
            raise ValueError(f'SPPUNetNeck: feature shapes {got} do not double from f2 to img '
                             '(expected [3, H, W], [64, H/2, W/2], [128, H/4, W/4] x 3)')
        h4, w4 = h // 4, w // 4
        if (h4 // 64) * (w4 // 64) < 2:
            raise ValueError(f'SPPUNetNeck: the 64x64 average pool of f4 ({h4} x {w4}) leaves '
                             f'{(h4 // 64) * (w4 // 64)} cells; the reference needs at least 2 '
                             '(AvgPool2d / GroupNorm)')

    def forward(self, feats):
        self.check_shapes(feats)
        for i, f in enumerate(feats):
            _check_cuda(f, f'feats[{i}]')
        self._forward_only(*feats)
        b, _, h, w = feats[0].shape
        L = capi.lib()
        key = (h, w, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            hd = ctypes.c_void_p()
            capi.check(L.dfm_spp_neck_create(h, w, _IMPL[self.conv_impl], ctypes.byref(hd)),
                       'dfm_spp_neck_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_spp_neck_set_param(self._handle, k, p, m),
            f'dfm_spp_neck_set_param({k.decode()})'))
        feats = [f.contiguous() for f in feats]
        dev = feats[0].device
        stereo = torch.empty((b, 32, h, w), device=dev)
        sem = torch.empty((b, 32, h // 4, w // 4), device=dev)
        cl = torch.empty((h, w, 32), device=dev) if b == 1 else None
        for i in range(b):
            capi.check(L.dfm_spp_neck_forward(
                self._handle, *[_ptr(f[i]) for f in feats], _ptr(cl), _ptr(stereo[i]),
                _ptr(sem[i]), _stream()), 'dfm_spp_neck_forward')
        if cl is not None:
            stereo._dfm_cl = cl
        return stereo, sem

    def debug_tensor(self, name, shape):
        """Channels-last intermediate of the last forward: raw conv outputs 'conv0', 'redir0',
        'conv1', 'rpn0', 'rpn1', 'lastconv'; 'pool64' .. 'pool8', 'spp64' .. 'spp8', 'concat',
        'x0', 'x1' (tests only)."""
        return _debug_tensor(self._handle, 'dfm_spp_neck_debug_tensor', name, shape)


@BACKBONES.register_module()
class BEVHourglass(_HandleMirror):
    """Drop-in for the reference ``BEVHourglass`` forward with GroupNorm
    (backbones/bev_hourglass.py:11-137; ``backbone_3d`` of
    configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:146-150).  The SyncBN variant is the frozen
    LiDAR teacher's (config :30-36, training only) and is not mirrored."""
    _destroy = 'dfm_bev_hourglass_destroy'

    def __init__(self, in_channels, out_channels, norm_cfg=None, output_prehg_feat=True,
                 conv_impl='auto'):
        super().__init__()
        assert norm_cfg is not None and norm_cfg.get('type') == 'GN' and \
            norm_cfg.get('num_groups', 32) == 32, 'only the GroupNorm(32) variant is implemented'
        self.out_channels = out_channels
        self.norm_cfg = norm_cfg
        self.output_prehg_feat = output_prehg_feat
        self.in_channels = in_channels
        self.conv_impl = conv_impl
        self.compress_conv = _ConvGN2d(in_channels, out_channels)
        self.bev_hourglass = _Hourglass2d(out_channels)
        self.num_bev_features = out_channels
        self._handle = None
        self._key = None

    def forward(self, spatial_features):
        _check_cuda(spatial_features, 'spatial_features')
        self._forward_only(spatial_features)
        b, c, ny, nx = spatial_features.shape
        assert c == self.in_channels
        L = capi.lib()
        key = (ny, nx, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            desc = capi.BevDesc(self.in_channels, self.out_channels, ny, nx,
                                _IMPL[self.conv_impl])
            hd = ctypes.c_void_p()
            capi.check(L.dfm_bev_hourglass_create(ctypes.byref(desc), ctypes.byref(hd)),
                       'dfm_bev_hourglass_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_bev_hourglass_set_param(self._handle, k, p, m),
            f'dfm_bev_hourglass_set_param({k.decode()})'))
        x = spatial_features.contiguous()
        out = torch.empty((b, self.out_channels, ny, nx), device=x.device)
        pre = torch.empty_like(out) if self.output_prehg_feat else None
        for i in range(b):
            capi.check(L.dfm_bev_hourglass_forward(
                self._handle, _ptr(x[i]), _ptr(pre[i]) if pre is not None else None,
                _ptr(out[i]), _stream()), 'dfm_bev_hourglass_forward')
        return (pre, out) if self.output_prehg_feat else out   # bev_hourglass.py:46-50

    def debug_tensor(self, name, shape):
        """Raw output [H, W, C] of 'compress' or 'conv1' .. 'conv6' (tests only)."""
        return _debug_tensor(self._handle, 'dfm_bev_hourglass_debug_tensor', name, shape)


@HEADS.register_module()
class LIGAAnchor3DHead(_HandleMirror):
    """Forward of the reference ``LIGAAnchor3DHead`` (dense_heads/liga_anchor3d_head.py:
    12-128): ``forward(feats) -> ([cls_score], [bbox_pred], [dir_cls_preds])``.  Anchor
    generation, target assignment, losses and ``get_bboxes`` (NMS) stay with the reference's
    PyTorch code (SURVEY.md section 2.1: heads only consume the hot path's output); the
    constructor keeps their arguments so the config block builds unchanged."""
    _destroy = 'dfm_anchor_head_destroy'

    def __init__(self, num_classes, in_channels, feat_channels=256, num_convs=2,
                 norm_cfg=None, use_direction_classifier=True,
                 anchor_generator=dict(type='Anchor3DRangeGenerator',
                                       sizes=[[3.9, 1.6, 1.56]], rotations=[0, 1.57]),
                 bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'), normalizer_clamp_value=10,
                 reduce_avg_factor=True, train_cfg=None, test_cfg=None, conv_impl='auto',
                 **kwargs):
        super().__init__()
        assert norm_cfg is not None and norm_cfg.get('type') == 'GN' and \
            norm_cfg.get('num_groups', 32) == 32, 'only the GroupNorm(32) variant is implemented'
        self.num_classes, self.in_channels = num_classes, in_channels
        self.feat_channels, self.num_convs = feat_channels, num_convs
        self.norm_cfg = norm_cfg
        self.use_direction_classifier = use_direction_classifier
        self.normalizer_clamp_value = normalizer_clamp_value
        self.reduce_avg_factor = reduce_avg_factor
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.extra_cfg = dict(anchor_generator=anchor_generator, bbox_coder=bbox_coder, **kwargs)
        # Anchor3DRangeGenerator.num_base_anchors (core/anchor/anchor_3d_generator.py:78-82)
        sizes = np.asarray(anchor_generator.get('sizes', [[3.9, 1.6, 1.56]])).reshape(-1, 3)
        self.num_anchors = len(anchor_generator.get('rotations', [0, 1.5707963])) * len(sizes)
        self.box_code_size = int(bbox_coder.get('code_size', 7))   # DeltaXYZWLHRBBoxCoder
        self.conv_impl = conv_impl
        # _init_layers (:37-75)
        self.cls_convs = nn.Sequential(*[_ConvGN2d(in_channels if i == 0 else feat_channels,
                                                   feat_channels) for i in range(num_convs)])
        self.reg_convs = nn.Sequential(*[_ConvGN2d(in_channels if i == 0 else feat_channels,
                                                   feat_channels) for i in range(num_convs)])
        self.cls_out_channels = self.num_anchors * num_classes
        self.conv_cls = nn.Conv2d(feat_channels, self.cls_out_channels, 3, 1, 1)
        self.conv_reg = nn.Conv2d(feat_channels, self.num_anchors * self.box_code_size, 3, 1, 1)
        if use_direction_classifier:
            self.conv_dir_cls = nn.Conv2d(feat_channels, self.num_anchors * 2, 1)
        self._handle = None
        self._key = None

    def forward(self, feats):
        if not isinstance(feats, list):                      # :104-105
            feats = [feats]
        outs = [self.forward_single(x) for x in feats]       # multi_apply
        return tuple(map(list, zip(*outs)))

    def forward_single(self, x):
        _check_cuda(x, 'x')
        self._forward_only(x)
        b, c, ny, nx = x.shape
        assert c == self.in_channels
        L = capi.lib()
        nd = self.num_anchors * 2 if self.use_direction_classifier else 0
        key = (ny, nx, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            desc = capi.AnchorHeadDesc(
                self.in_channels, self.feat_channels, self.num_convs, self.cls_out_channels,
                self.num_anchors * self.box_code_size, nd, ny, nx, _IMPL[self.conv_impl])
            hd = ctypes.c_void_p()
            capi.check(L.dfm_anchor_head_create(ctypes.byref(desc), ctypes.byref(hd)),
                       'dfm_anchor_head_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_anchor_head_set_param(self._handle, k, p, m),
            f'dfm_anchor_head_set_param({k.decode()})'))
        x = x.contiguous()
        cls = torch.empty((b, self.cls_out_channels, ny, nx), device=x.device)
        box = torch.empty((b, self.num_anchors * self.box_code_size, ny, nx), device=x.device)
        dirc = torch.empty((b, nd, ny, nx), device=x.device) if nd else None
        for i in range(b):
            capi.check(L.dfm_anchor_head_forward(
                self._handle, _ptr(x[i]), _ptr(cls[i]), _ptr(box[i]),
                _ptr(dirc[i]) if dirc is not None else None, _stream()),
                'dfm_anchor_head_forward')
        return cls, box, dirc

    def debug_tensor(self, name, shape):
        """Raw output [ny, nx, C] of 'cls<i>' / 'reg<i>' or of the output convs 'cls_out'
        (cls + dir channels) / 'reg_out', at their widths padded to 32 (tests only)."""
        return _debug_tensor(self._handle, 'dfm_anchor_head_debug_tensor', name, shape)


@HEADS.register_module()
class Anchor3DHead(_HandleMirror):
    """Forward of the reference ``Anchor3DHead`` (dense_heads/anchor3d_head.py:15-185), the
    ``bbox_head_3d`` of both MultiViewDfM (Waymo) configs: ``forward(feats) -> ([cls_score],
    [bbox_pred], [dir_cls_preds or None])``.  The three 1x1 convs run as one tensor-core GEMM
    that reads the BEV map once (``csrc/head1x1_tc.cuh``).  Anchor generation, target
    assignment, losses and ``get_bboxes`` (NMS) stay with the reference's PyTorch code; the
    constructor keeps their arguments so the config block builds unchanged, and the
    ``state_dict`` (``conv_cls`` / ``conv_reg`` / ``conv_dir_cls``) is the reference's."""
    _destroy = 'dfm_anchor3d_head_destroy'

    def __init__(self, num_classes, in_channels, train_cfg=None, test_cfg=None,
                 feat_channels=256, use_direction_classifier=True,
                 anchor_generator=dict(type='Anchor3DRangeGenerator',
                                       range=[0, -39.68, -1.78, 69.12, 39.68, -1.78],
                                       strides=[2], sizes=[[3.9, 1.6, 1.56]],
                                       rotations=[0, 1.57], custom_values=[],
                                       reshape_out=False),
                 assigner_per_size=False, assign_per_class=False, diff_rad_by_sin=True,
                 dir_offset=-np.pi / 2, dir_limit_offset=0,
                 bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'),
                 loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=2.0),
                 loss_dir=dict(type='CrossEntropyLoss', loss_weight=0.2), loss_iou=None,
                 init_cfg=None, conv_impl='auto'):
        super().__init__()
        self.in_channels, self.num_classes = in_channels, num_classes
        self.feat_channels = feat_channels
        self.diff_rad_by_sin = diff_rad_by_sin
        self.use_direction_classifier = use_direction_classifier
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.assigner_per_size, self.assign_per_class = assigner_per_size, assign_per_class
        self.dir_offset, self.dir_limit_offset = dir_offset, dir_limit_offset
        self.init_cfg = init_cfg
        self.extra_cfg = dict(anchor_generator=anchor_generator, bbox_coder=bbox_coder,
                              loss_cls=loss_cls, loss_bbox=loss_bbox, loss_dir=loss_dir,
                              loss_iou=loss_iou)
        # Anchor3DRangeGenerator.num_base_anchors (core/anchor/anchor_3d_generator.py:78-82)
        sizes = np.asarray(anchor_generator.get('sizes', [[3.9, 1.6, 1.56]])).reshape(-1, 3)
        self.num_anchors = len(anchor_generator.get('rotations', [0, 1.5707963])) * len(sizes)
        self.box_code_size = int(bbox_coder.get('code_size', 7))   # DeltaXYZWLHRBBoxCoder
        self.use_sigmoid_cls = loss_cls.get('use_sigmoid', False)  # anchor3d_head.py:99-102
        if not self.use_sigmoid_cls:
            self.num_classes += 1
        self.conv_impl = conv_impl
        # _init_layers (:139-147): 1x1 convs on feat_channels (in_channels is not used)
        self.cls_out_channels = self.num_anchors * self.num_classes
        self.conv_cls = nn.Conv2d(feat_channels, self.cls_out_channels, 1)
        self.conv_reg = nn.Conv2d(feat_channels, self.num_anchors * self.box_code_size, 1)
        if use_direction_classifier:
            self.conv_dir_cls = nn.Conv2d(feat_channels, self.num_anchors * 2, 1)
        self._handle = None
        self._key = None

    def forward(self, feats):
        outs = [self.forward_single(x) for x in feats]       # multi_apply (:166-185)
        return tuple(map(list, zip(*outs)))

    def forward_single(self, x):
        _check_cuda(x, 'x')
        self._forward_only(x)
        b, c, ny, nx = x.shape
        if c != self.feat_channels:
            raise RuntimeError(f'Anchor3DHead: input has {c} channels, the convs take '
                               f'feat_channels = {self.feat_channels}')
        L = capi.lib()
        nd = self.num_anchors * 2 if self.use_direction_classifier else 0
        nr = self.num_anchors * self.box_code_size
        key = (ny, nx, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            desc = capi.Anchor3DHeadDesc(self.feat_channels, self.cls_out_channels, nr, nd,
                                         ny, nx, _IMPL[self.conv_impl])
            hd = ctypes.c_void_p()
            capi.check(L.dfm_anchor3d_head_create(ctypes.byref(desc), ctypes.byref(hd)),
                       'dfm_anchor3d_head_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_anchor3d_head_set_param(self._handle, k, p, m),
            f'dfm_anchor3d_head_set_param({k.decode()})'))
        x = x.contiguous()
        cls = torch.empty((b, self.cls_out_channels, ny, nx), device=x.device)
        box = torch.empty((b, nr, ny, nx), device=x.device)
        dirc = torch.empty((b, nd, ny, nx), device=x.device) if nd else None
        for i in range(b):
            capi.check(L.dfm_anchor3d_head_forward(
                self._handle, _ptr(x[i]), _ptr(cls[i]), _ptr(box[i]),
                _ptr(dirc[i]) if dirc is not None else None, _stream()),
                'dfm_anchor3d_head_forward')
        return cls, box, dirc


class _ConvModuleConv(nn.Module):
    """Parameter layout of mmcv ConvModule without norm or activation: .conv only."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, padding=k // 2)


@NECKS.register_module()
class FPN(_HandleMirror):
    """mmdet's ``FPN`` image neck in the configuration of both MultiViewDfM (Waymo) configs
    (``neck``: in_channels [256, 512, 1024, 2048], out_channels 64, num_outs 4) on CUDA
    (``csrc/fpn_api.inc``): lateral 1x1 convs with the nearest-upsampled top-down merge fused
    into one tensor-core GEMM per level, then the 3x3 ``fpn_convs``.  ``forward(inputs) ->
    tuple`` of 4 NCHW maps, for any batch size in one call.  The ``state_dict`` is mmdet's
    (``lateral_convs.{0..3}.conv.*``, ``fpn_convs.{0..3}.conv.*``).  Only that configuration is
    implemented: extra convs, norm, activation, non-nearest upsampling, ``start_level != 0`` and
    ``num_outs`` other than the number of levels raise ``NotImplementedError``.  It is
    registered in the local ``NECKS`` only: KITTI's ``neck_2d`` is also an mmdet ``FPN`` (with
    extra convs) and must keep resolving to mmdet's class.
    Patch: ``model.neck = FPN(**cfg.model.neck)``."""
    _destroy = 'dfm_fpn_destroy'

    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1,
                 add_extra_convs=False, relu_before_extra_convs=False, no_norm_on_lateral=False,
                 conv_cfg=None, norm_cfg=None, act_cfg=None, upsample_cfg=dict(mode='nearest'),
                 init_cfg=None, conv_impl='auto'):
        super().__init__()
        in_channels = list(in_channels)
        n = len(in_channels)
        if n != 4:
            raise NotImplementedError(f'FPN: {n} input levels; only 4 are implemented')
        if start_level != 0 or end_level not in (-1, n - 1):
            raise NotImplementedError('FPN: only start_level=0 and end_level=-1 are implemented')
        if num_outs < n:
            raise ValueError(f'FPN: num_outs = {num_outs} is below the {n} input levels')
        if num_outs > n or add_extra_convs:
            raise NotImplementedError('FPN: extra levels (num_outs > number of inputs, '
                                      'add_extra_convs) are not implemented')
        if conv_cfg is not None or norm_cfg is not None or act_cfg is not None:
            raise NotImplementedError('FPN: conv_cfg, norm_cfg and act_cfg must be None')
        up = dict(upsample_cfg or {})
        if up.get('mode', 'nearest') != 'nearest' or set(up) - {'mode'}:
            raise NotImplementedError("FPN: only upsample_cfg=dict(mode='nearest') is implemented")
        if any(c % 16 for c in in_channels + [out_channels]):
            raise NotImplementedError('FPN: channel counts must be multiples of 16')
        if out_channels not in (32, 64):
            raise NotImplementedError('FPN: out_channels must be 64 (tensor cores) or 32')
        self.in_channels, self.out_channels = in_channels, out_channels
        self.num_ins, self.num_outs = n, num_outs
        self.start_level, self.backbone_end_level = 0, n
        self.add_extra_convs = False
        self.relu_before_extra_convs = relu_before_extra_convs
        self.no_norm_on_lateral = no_norm_on_lateral
        self.upsample_cfg = up
        self.init_cfg = init_cfg
        self.conv_impl = conv_impl
        self.lateral_convs = nn.ModuleList(_ConvModuleConv(c, out_channels, 1)
                                           for c in in_channels)
        self.fpn_convs = nn.ModuleList(_ConvModuleConv(out_channels, out_channels, 3)
                                       for _ in in_channels)
        self._handle = None
        self._key = None

    def check_shapes(self, inputs):
        """Raises ValueError on inputs that disagree with the constructor."""
        if len(inputs) != self.num_ins:
            raise ValueError(f'FPN takes {self.num_ins} feature maps, got {len(inputs)}')
        for i, (x, c) in enumerate(zip(inputs, self.in_channels)):
            if x.dim() != 4 or x.shape[1] != c or x.shape[0] != inputs[0].shape[0]:
                raise ValueError(f'FPN: inputs[{i}] has shape {tuple(x.shape)}; expected '
                                 f'[{inputs[0].shape[0]}, {c}, H, W]')

    def forward(self, inputs):
        self.check_shapes(inputs)
        for i, x in enumerate(inputs):
            _check_cuda(x, f'inputs[{i}]')
        self._forward_only(*inputs)
        b = inputs[0].shape[0]
        sizes = [tuple(x.shape[2:]) for x in inputs]
        dev = inputs[0].device
        outs = tuple(torch.empty((b, self.out_channels) + s, device=dev) for s in sizes)
        if b == 0:
            return outs
        L = capi.lib()
        key = (b, tuple(sizes), self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            desc = capi.FpnDesc()
            desc.in_channels[:] = self.in_channels
            desc.out_channels = self.out_channels
            desc.level_h[:] = [s[0] for s in sizes]
            desc.level_w[:] = [s[1] for s in sizes]
            desc.num_images, desc.conv_impl = b, _IMPL[self.conv_impl]
            hd = ctypes.c_void_p()
            capi.check(L.dfm_fpn_create(ctypes.byref(desc), ctypes.byref(hd)), 'dfm_fpn_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_fpn_set_param(self._handle, k, p, m), f'dfm_fpn_set_param({k.decode()})'))
        xs = [x.contiguous() for x in inputs]
        arr = ctypes.c_void_p * 4
        capi.check(L.dfm_fpn_forward(self._handle, arr(*[x.data_ptr() for x in xs]),
                                     arr(*[o.data_ptr() for o in outs]), _stream()),
                   'dfm_fpn_forward')
        return outs

    def debug_tensor(self, name, shape):
        """Channels-last [B, H, W, C] intermediate of the last forward: the merged laterals
        'merged0' .. 'merged3' and the raw fpn_conv outputs before the bias 'fpn0' .. 'fpn3'
        (tests only)."""
        return _debug_tensor(self._handle, 'dfm_fpn_debug_tensor', name, shape)


class _LigaBasicBlock(nn.Module):
    """Parameter layout of the reference ``LigaBasicBlock`` (backbones/liga_resnet.py:11-54):
    conv1 / bn1 / conv2 / bn2 and an optional ``downsample`` = (1x1 conv, BatchNorm)."""

    def __init__(self, inplanes, planes, stride, dilation, downsample):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, dilation, dilation, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = nn.Sequential(
            nn.Conv2d(inplanes, planes, 1, stride, bias=False),
            nn.BatchNorm2d(planes)) if downsample else None
        self.stride, self.dilation = stride, dilation


@BACKBONES.register_module()
class LIGAResNet(_HandleMirror):
    """The reference ``LIGAResNet`` (backbones/liga_resnet.py) in the configuration of the shipped
    KITTI config's ``backbone`` on CUDA (``csrc/liga_resnet_api.inc``): depth 34, strides
    (1, 2, 1, 1), dilations (1, 1, 2, 4), num_channels_factor (1, 2, 2, 2), no max-pool and no
    ReLU after the residual adds.  ``forward(img [B, 3, H, W]) -> tuple`` of 4 NCHW maps
    ([B, 64, H2, W2] and three [B, 128, H4, W4], H2 = ceil(H / 2), H4 = ceil(H2 / 2)) for any
    batch size in one C call.  The ``state_dict`` is the reference's (204 entries, BatchNorm
    running statistics included); BatchNorm runs in eval form.  Other depths, strides,
    dilations or channel factors, ``with_max_pool``, ``block_with_final_relu``, ``deep_stem``,
    ``avg_down``, ``dcn``, ``plugins`` and non-BN norms raise ``NotImplementedError``.  It is
    registered in the local ``BACKBONES`` only (forward-only: training keeps mmdet3d's class).
    Patch: ``model.backbone = LIGAResNet(**cfg.model.backbone)``."""
    _destroy = 'dfm_liga_resnet_destroy'
    STAGE_BLOCKS = (3, 4, 6, 3)

    def __init__(self, depth, in_channels=3, stem_channels=None, base_channels=64, num_stages=4,
                 strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3),
                 style='pytorch', deep_stem=False, avg_down=False, frozen_stages=-1,
                 conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), norm_eval=True,
                 dcn=None, stage_with_dcn=(False, False, False, False), plugins=None,
                 with_cp=False, zero_init_residual=True, init_cfg=None, with_max_pool=True,
                 block_with_final_relu=True, num_channels_factor=None, conv_impl='auto'):
        super().__init__()
        checks = (
            (depth == 34, f'depth={depth}'),
            (in_channels == 3 and stem_channels in (None, 64) and base_channels == 64,
             'in_channels / stem_channels / base_channels other than 3 / 64 / 64'),
            (num_stages == 4 and tuple(strides) == (1, 2, 1, 1) and
             tuple(dilations) == (1, 1, 2, 4), f'strides={strides}, dilations={dilations}'),
            (tuple(out_indices) == (0, 1, 2, 3), f'out_indices={out_indices}'),
            (num_channels_factor is not None and tuple(num_channels_factor) == (1, 2, 2, 2),
             f'num_channels_factor={num_channels_factor}'),
            (style == 'pytorch', f'style={style!r}'),
            (not deep_stem, 'deep_stem'), (not avg_down, 'avg_down'),
            (dcn is None and not any(stage_with_dcn), 'dcn'), (plugins is None, 'plugins'),
            (conv_cfg is None, 'conv_cfg'),
            (norm_cfg is not None and norm_cfg.get('type') in ('BN', 'SyncBN'),
             f'norm_cfg={norm_cfg}'),
            (not with_max_pool, 'with_max_pool'),
            (not block_with_final_relu, 'block_with_final_relu'))
        for ok, what in checks:
            if not ok:
                raise NotImplementedError(
                    f'LIGAResNet: {what} is not implemented (only the shipped KITTI backbone: '
                    'depth 34, strides (1, 2, 1, 1), dilations (1, 1, 2, 4), channel factors '
                    '(1, 2, 2, 2), no max-pool, no final block ReLU, BatchNorm)')
        self.depth, self.num_stages = depth, num_stages
        self.strides, self.dilations = tuple(strides), tuple(dilations)
        self.out_indices, self.style = tuple(out_indices), style
        self.frozen_stages, self.norm_cfg, self.norm_eval = frozen_stages, norm_cfg, norm_eval
        self.with_cp, self.zero_init_residual, self.init_cfg = with_cp, zero_init_residual, init_cfg
        self.with_max_pool, self.block_with_final_relu = False, False
        self.num_channels_factor = tuple(num_channels_factor)
        self.conv_impl = conv_impl
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.res_layers = []
        inplanes = 64
        for i, n in enumerate(self.STAGE_BLOCKS):
            planes = 64 * self.num_channels_factor[i]
            blocks = []
            for j in range(n):
                stride = self.strides[i] if j == 0 else 1
                blocks.append(_LigaBasicBlock(inplanes, planes, stride, self.dilations[i],
                                              j == 0 and (stride != 1 or inplanes != planes)))
                inplanes = planes
            self.add_module(f'layer{i + 1}', nn.Sequential(*blocks))
            self.res_layers.append(f'layer{i + 1}')
        self._handle = None
        self._key = None

    @staticmethod
    def output_sizes(h, w):
        """(H2, W2), (H4, W4): PyTorch's output-size rule of the stride-2 convs."""
        h2, w2 = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        return (h2, w2), ((h2 - 1) // 2 + 1, (w2 - 1) // 2 + 1)

    @staticmethod
    def check_shapes(img):
        """Raises ValueError on an input that is not [B, 3, H, W] with a non-empty image."""
        if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[1] != 3 or \
                img.shape[2] < 1 or img.shape[3] < 1:
            shape = tuple(img.shape) if isinstance(img, torch.Tensor) else type(img).__name__
            raise ValueError(f'LIGAResNet takes an image batch [B, 3, H, W], got {shape}')

    def forward(self, img):
        self.check_shapes(img)
        _check_cuda(img, 'img')
        self._forward_only(img)
        b, _, h, w = img.shape
        (h2, w2), (h4, w4) = self.output_sizes(h, w)
        dev = img.device
        outs = (torch.empty((b, 64, h2, w2), device=dev),) + \
            tuple(torch.empty((b, 128, h4, w4), device=dev) for _ in range(3))
        if b == 0:
            return outs
        L = capi.lib()
        key = (b, h, w, self.conv_impl)
        if self._handle is None or key != self._key:
            self.release()
            desc = capi.LigaResNetDesc(h, w, b, _IMPL[self.conv_impl])
            hd = ctypes.c_void_p()
            capi.check(L.dfm_liga_resnet_create(ctypes.byref(desc), ctypes.byref(hd)),
                       'dfm_liga_resnet_create')
            self._handle, self._key = hd, key
            self._sync = _ParamSync()
        self._sync.sync(self, lambda k, p, m: capi.check(
            L.dfm_liga_resnet_set_param(self._handle, k, p, m),
            f'dfm_liga_resnet_set_param({k.decode()})'))
        x = img.contiguous()
        arr = ctypes.c_void_p * 4
        capi.check(L.dfm_liga_resnet_forward(self._handle, _ptr(x),
                                             arr(*[o.data_ptr() for o in outs]), _stream()),
                   'dfm_liga_resnet_forward')
        return outs

    def debug_tensor(self, name, shape):
        """Channels-last [B, h, w, C] intermediate of the last forward: 'stem' (raw conv1),
        'layerI.J.conv1' / 'layerI.J.conv2' / 'layer2.0.downsample' (raw conv outputs) and the
        block outputs 'layerI.J' (tests only)."""
        return _debug_tensor(self._handle, 'dfm_liga_resnet_debug_tensor', name, shape)


def aligned_voxel_centers(n_voxels, voxel_range):
    """Per-axis voxel-centre coordinates exactly as
    AlignedAnchor3DRangeGenerator.anchors_single_range computes them
    (core/anchor/anchor_3d_generator.py:283-310, align_corner=False)."""
    nx, ny, nz = n_voxels
    r = torch.tensor(voxel_range, dtype=torch.float32)
    out = []
    for lo, hi, n in ((r[0], r[3], nx), (r[1], r[4], ny), (r[2], r[5], nz)):
        c = torch.linspace(lo, hi, n + 1)
        c = c + (c[1] - c[0]) / 2
        out.append(c[:n].contiguous())
    return out


def _require_identity_3d_aug(img_meta):
    """point_sample first undoes the 3-D augmentation recorded in img_meta
    (apply_3d_transformation(reverse=True), coord_transform.py:9-92).  At test time the
    keys are absent or identity; the lifting kernel does not implement the reverse
    transform, so anything else must fail loudly rather than lift with wrong points."""
    rot = img_meta.get('pcd_rotation')
    if rot is not None and not np.allclose(np.asarray(rot, dtype=np.float64), np.eye(3)):
        raise NotImplementedError('multiview_lift: non-identity pcd_rotation')
    scale = img_meta.get('pcd_scale_factor', 1.0)
    if not np.isclose(float(scale), 1.0):
        raise NotImplementedError('multiview_lift: pcd_scale_factor != 1')
    trans = img_meta.get('pcd_trans')
    if trans is not None and np.any(np.asarray(trans, dtype=np.float64) != 0):
        raise NotImplementedError('multiview_lift: non-zero pcd_trans')
    if img_meta.get('pcd_horizontal_flip', False) or img_meta.get('pcd_vertical_flip', False):
        raise NotImplementedError('multiview_lift: pcd flip')


def multiview_lift(feats, img_meta, n_voxels, voxel_range, num_views,
                   num_frames, temporal_aggregate='mean', out=None, channels_last=True):
    """The lifting loop of MultiViewDfM.feature_transformation
    (multiview_dfm.py:139-209, valid_sample=True) for one sample.
    feats: [T*Nv, C, Hf, Wf] CUDA -> [C(*T), Nx, Ny, Nz].  The returned tensor has the
    reference's shape but channels-last strides (memory [Nx, Ny, Nz, C]): that is what the
    necks' conv loaders read, so neither the lifting kernel's stores nor the neck pay for a
    layout change.  ``out``: optional contiguous [Nx, Ny, Nz, C(*T)] CUDA buffer to fill.
    ``channels_last=False`` runs the reference-layout kernel (contiguous [C, Nx, Ny, Nz])."""
    _check_cuda(feats, 'feats')
    s, c, hf, wf = feats.shape
    assert s == num_views * num_frames
    _require_identity_3d_aug(img_meta)
    sf = img_meta.get('scale_factor', 1.0)
    sf = np.atleast_1d(np.asarray(sf, dtype=np.float32))
    sx, sy = (float(sf[0]), float(sf[1])) if sf.size >= 2 else (float(sf[0]),) * 2
    crop = img_meta.get('img_crop_offset', (0.0, 0.0))
    if np.isscalar(crop):
        crop = (crop, crop)
    desc = capi.LiftDesc()
    desc.num_frames, desc.num_views, desc.channels = num_frames, num_views, c
    desc.feat_h, desc.feat_w = hf, wf
    desc.n_voxels[:] = list(n_voxels)
    desc.scale_x, desc.scale_y = sx, sy
    desc.crop_x, desc.crop_y = float(crop[0]), float(crop[1])
    desc.flip = int(bool(img_meta.get('flip', False)))
    desc.input_h, desc.input_w = img_meta['input_shape'][:2]
    desc.concat = int(temporal_aggregate == 'concat')
    # the reference converts ori_lidar2img to the feature dtype (fp32) first
    proj = np.asarray(img_meta['ori_lidar2img'], dtype=np.float32)[:s]
    proj = np.ascontiguousarray(proj.astype(np.float64).reshape(s, 16))
    img_w = np.ascontiguousarray(
        [int(img_meta['img_shape'][i][1]) for i in range(s)], dtype=np.int32)
    xs, ys, zs = aligned_voxel_centers(n_voxels, voxel_range)
    cout = c * num_frames if desc.concat else c
    if not channels_last:
        assert out is None
        vol = torch.empty((cout, n_voxels[0], n_voxels[1], n_voxels[2]),
                          device=feats.device, dtype=torch.float32)
        capi.check(capi.lib().dfm_multiview_lift(
            ctypes.byref(desc), _ptr(feats.contiguous()),
            proj.ctypes.data_as(ctypes.c_void_p),
            img_w.ctypes.data_as(ctypes.c_void_p),
            ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(ys.data_ptr()),
            ctypes.c_void_p(zs.data_ptr()), _ptr(vol), _stream()),
            'dfm_multiview_lift')
        return vol
    shape_cl = (n_voxels[0], n_voxels[1], n_voxels[2], cout)
    if out is None:
        out = torch.empty(shape_cl, device=feats.device, dtype=torch.float32)
    assert tuple(out.shape) == shape_cl and out.is_contiguous() and out.is_cuda
    capi.check(capi.lib().dfm_multiview_lift_cl(
        ctypes.byref(desc), _ptr(feats.contiguous()),
        proj.ctypes.data_as(ctypes.c_void_p),
        img_w.ctypes.data_as(ctypes.c_void_p),
        ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(ys.data_ptr()),
        ctypes.c_void_p(zs.data_ptr()), _ptr(out), _stream()),
        'dfm_multiview_lift_cl')
    return out.permute(3, 0, 1, 2)


def voxel_sample(voxel_features, voxel_range, voxel_size, depth_samples, proj_mat,
                 downsample_factor, img_scale_factor, img_crop_offset, img_flip,
                 img_pad_shape, img_shape, aligned=True, padding_mode='zeros',
                 align_corners=True):
    """Same signature as the reference ``voxel_sample``
    (fusion_layers/point_fusion.py:324-339): [1, C, Nx, Ny, Nz] CUDA voxel features ->
    [1, C, D, H, W] frustum features (D = len(depth_samples[::downsample_factor]))."""
    _check_cuda(voxel_features, 'voxel_features')
    if padding_mode != 'zeros' or not align_corners:
        raise NotImplementedError("voxel_sample: only padding_mode='zeros', "
                                  'align_corners=True (the reference defaults)')
    n, c, nx, ny, nz = voxel_features.shape
    assert n == 1
    h, w = img_pad_shape[:2]
    ho, wo = round(h / downsample_factor), round(w / downsample_factor)
    depths = torch.as_tensor(depth_samples, dtype=torch.float32).detach().cpu()[
        ::downsample_factor].contiguous()
    sf = np.atleast_1d(np.asarray(
        img_scale_factor.detach().cpu() if isinstance(img_scale_factor, torch.Tensor)
        else img_scale_factor, dtype=np.float32))
    crop = np.atleast_1d(np.asarray(
        img_crop_offset.detach().cpu() if isinstance(img_crop_offset, torch.Tensor)
        else img_crop_offset, dtype=np.float32))
    desc = capi.VoxelSampleDesc()
    desc.channels, desc.nx, desc.ny, desc.nz = c, nx, ny, nz
    desc.voxel_range[:] = [float(v) for v in voxel_range]
    desc.voxel_size[:] = [float(v) for v in voxel_size]
    desc.num_depths, desc.out_h, desc.out_w = depths.numel(), ho, wo
    desc.downsample_factor = int(downsample_factor)
    desc.scale_x, desc.scale_y = float(sf[0]), float(sf[-1] if sf.size > 1 else sf[0])
    desc.crop_x, desc.crop_y = float(crop[0]), float(crop[-1] if crop.size > 1 else crop[0])
    desc.flip, desc.img_w = int(bool(img_flip)), int(img_shape[1])
    desc.aligned = int(bool(aligned))
    pm = np.asarray(proj_mat.detach().cpu() if isinstance(proj_mat, torch.Tensor) else proj_mat,
                    dtype=np.float64)
    pad = np.eye(4)
    pad[:pm.shape[0], :pm.shape[1]] = pm
    P = (ctypes.c_double * 16)(*pad.reshape(-1).tolist())
    out = torch.empty((1, c, depths.numel(), ho, wo), device=voxel_features.device)
    capi.check(capi.lib().dfm_voxel_sample(
        ctypes.byref(desc), _ptr(voxel_features.contiguous()),
        ctypes.c_void_p(depths.data_ptr()), P, _ptr(out), _stream()), 'dfm_voxel_sample')
    return out


class MultiViewDfMFeatureTransformation:
    """Method-override mix-in for the reference detector: same signature, same
    ``img_metas`` keys and same return tuple as
    ``MultiViewDfM.feature_transformation`` (detectors/multiview_dfm.py:119-268)
    for the shipped Waymo configs (``valid_sample=True``, no ``backbone_3d``, no
    ``depth_head``: configs/dfm/multiview-dfm_r101_dcn_2x16_waymoD5-3d-3class_camsync
    [_10sweeps].py:26-32).  Usage::

        class MultiViewDfMB200(MultiViewDfMFeatureTransformation, MultiViewDfM):
            pass

    The host object supplies what the reference reads from ``self``: ``n_voxels``,
    ``voxel_range`` (``anchor_generator['ranges'][0]``), ``temporal_aggregate``,
    ``valid_sample``, ``neck_3d`` (our ``OutdoorImVoxelNeck`` / ``DfMNeck``)."""

    def feature_transformation(self, batch_feats, img_metas, num_views, num_frames):
        if getattr(self, 'with_depth_head', False) or getattr(self, 'with_backbone_3d', False):
            raise NotImplementedError(
                'the CUDA feature_transformation covers the shipped configs '
                '(depth_head=None, backbone_3d=None); voxel_sample is not on that path')
        if not getattr(self, 'valid_sample', True):
            raise NotImplementedError('valid_sample=False is not implemented')
        nvx = list(self.n_voxels)
        cout = batch_feats[0].shape[1] * (num_frames if self.temporal_aggregate == 'concat' else 1)
        # one channels-last buffer for the batch; the reference-shaped view is returned
        buf = torch.empty((len(batch_feats), nvx[0], nvx[1], nvx[2], cout),
                          device=batch_feats[0].device, dtype=torch.float32)
        for b, (feature, img_meta) in enumerate(zip(batch_feats, img_metas)):   # :128
            meta = dict(img_meta)
            if 'scale_factor' not in meta:                           # :129-138
                meta['scale_factor'] = 1.0
            multiview_lift(feature, meta, nvx, list(self.voxel_range), num_views,
                           num_frames, self.temporal_aggregate, out=buf[b])
        volume_feat = buf.permute(0, 4, 1, 2, 3)                     # (B, C, Nx, Ny, Nz), :209
        if getattr(self, 'with_neck_3d', self.neck_3d is not None):
            volume_feat = self.neck_3d(volume_feat)[0]               # :263
        return (volume_feat, )                                       # :265-268
