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
    Anchor3DHead         mmdet3d/models/dense_heads/anchor3d_head.py:139-185, 407-547
                         (forward, get_bboxes; LIGAAnchor3DHead inherits the latter)
    SPPUNetNeck          mmdet3d/models/necks/spp_unet_neck.py (shipped KITTI config)
    FPN                  mmdet's FPN as the Waymo configs' image neck (mmdet 2.24 semantics)
    LIGAResNet           mmdet3d/models/backbones/liga_resnet.py (shipped KITTI config)
    ResNet               mmdet's ResNet-101 with DCNv2 as the Waymo configs' image backbone

The ``nn.Conv3d`` / ``nn.GroupNorm`` / ``nn.BatchNorm3d`` children below are
parameter containers only (they give the exact reference ``state_dict`` layout so
reference checkpoints load with ``strict=True``); their ``forward`` is never
called.  There is no PyTorch fallback: without the built library or an H100 the
modules raise.
"""
import collections
import copy
import ctypes
import itertools
import os

import numpy as np
import torch
import torch.nn as nn

from . import capi
from .registry import BACKBONES, DETECTORS, HEADS, NECKS

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
_UPLOADS = itertools.count(1)


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
        # a new value at every upload: the detectors' feature cache keeps the generation its
        # entries were computed under (``_ViewFeatureCache``)
        self.generation = 0
        self._watch = ()

    def mark_dirty(self):
        self._sig = None

    def pending(self):
        """True when the next ``sync`` will upload, found without building the ``state_dict``:
        ``mark_dirty`` was called, or a tensor of the last upload was replaced by another
        object, written in place (version) or moved (storage pointer)."""
        return self._sig is None or any(
            owner.get(k) is not t or t.data_ptr() != p or t._version != v
            for owner, k, t, p, v in self._watch)

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
        self.generation = next(_UPLOADS)
        self._watch = tuple((owner, k, v, v.data_ptr(), v._version)
                            for m in module.modules()
                            for owner in (m._parameters, m._buffers)
                            for k, v in owner.items() if v is not None)


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


class _HandleMirror(_CudaMirror):
    """A mirror that owns one handle of include/dfm_b200.h, of the family ``_family``
    (``dfm_<family>_create`` / ``_destroy`` / ``_set_param`` / ``_debug_tensor``).  Subclasses
    give the key the handle is built for, the create arguments and the forward."""
    _family = None
    _handle = None
    _key = None
    _batch = None

    def _ensure(self, key, create_args, batch=None):
        """``capi.lib()``, with a handle for ``key`` that holds the current parameters.  Another
        key destroys the handle and creates a new one, ``dfm_<family>_create(*create_args(),
        &handle)``, with a fresh ``_ParamSync``.  ``batch``, for the families with
        ``set_num_images``: another batch size alone keeps the handle and its uploads."""
        L = capi.lib()
        fn = f'dfm_{self._family}'
        if self._handle is not None and key == self._key:
            if batch is not None and batch != self._batch:
                capi.check(getattr(L, fn + '_set_num_images')(self._handle, batch),
                           fn + '_set_num_images')
                self._batch = batch
        else:
            self.release()
            hd = ctypes.c_void_p()
            capi.check(getattr(L, fn + '_create')(*create_args(), ctypes.byref(hd)),
                       fn + '_create')
            self._handle, self._key, self._batch = hd, key, batch
            self._sync = _ParamSync()
        set_param = getattr(L, fn + '_set_param')
        self._sync.sync(self, lambda k, p, n: capi.check(set_param(self._handle, k, p, n),
                                                         f'{fn}_set_param({k.decode()})'))
        return L

    def release(self):
        if self._handle is not None:
            getattr(capi.lib(), f'dfm_{self._family}_destroy')(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def init_weights(self):
        pass

    def debug_tensor(self, name, shape):
        """Channels-last copy of the intermediate ``name`` the handle's last forward wrote, through
        the test hook ``dfm_<family>_debug_tensor`` (shape must hold exactly that tensor; tests
        only).  The class docstring lists the names."""
        fn = f'dfm_{self._family}_debug_tensor'
        if self._handle is None:
            raise RuntimeError(f'{fn}: no forward has run')
        out = torch.empty(shape, device='cuda', dtype=torch.float32)
        capi.check(getattr(capi.lib(), fn)(self._handle, name.encode(), _ptr(out), out.numel(),
                                           _stream()), f'{fn}({name})')
        return out


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
class DfMBackbone(_HandleMirror):
    """Drop-in for the reference ``DfMBackbone`` (dfm_backbone.py:14-214).  Debug tensors
    (channels-last), each tower's 'raw0', 'cls3', 'raw1', 'c1' .. 'c6', 'cur', 'p0' and 'logit'
    ('<name>_mono' for the mono tower)."""
    _family = 'backbone'

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
        self._sync = _ParamSync()
        self._depth_sig = None

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

    def _prepare(self, h, w):
        def create_args():
            self._depth_sig = None   # a new handle has no depths
            return (ctypes.byref(capi.BackboneDesc(
                self.in_channels, self.cv_channels, h, w, self.num_planes,
                self.cost_sample_factor, int(self.feat_sample_factor), _IMPL[self.conv_impl])),)

        L = self._ensure((h, w, self.conv_impl), create_args)
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
        # stereo features that came out of our SPPUNetNeckTail carry a channels-last twin:
        # the plane-sweep loader reads it directly, no NCHW -> NHWC transposes
        cl_c = getattr(cur_stereo_feats, '_dfm_cl', None)
        cl_p = getattr(prev_stereo_feats, '_dfm_cl', None)
        if cl_c is not None and cl_p is not None and cl_c.shape == (h, w, c) == cl_p.shape:
            return self._forward_cl(cl_c, cl_p, img_metas)
        L = self._prepare(h, w)
        cur = cur_stereo_feats.contiguous()
        prev = prev_stereo_feats.contiguous()
        geom = geometry_from_meta(img_metas[0])
        cost, stereo, mono = self._outputs(h, w, cur.device)
        capi.check(L.dfm_backbone_forward(
            self._handle, _ptr(cur), _ptr(prev), ctypes.byref(geom), _ptr(cost),
            _ptr(stereo), _ptr(mono), _stream()), 'dfm_backbone_forward')
        return self._finish(cost, stereo, mono)

    def _outputs(self, h, w, dev):
        ho = round(h / self.cost_sample_factor)
        wo = round(w / self.cost_sample_factor)
        d = self.num_planes
        cost = torch.empty((1, 1, d, ho, wo), device=dev, dtype=torch.float32)
        stereo = torch.empty((1, self.cv_channels, d, ho, wo), device=dev,
                             dtype=torch.float32)
        return cost, stereo, torch.empty_like(stereo)

    def _forward_cl(self, cl_c, cl_p, img_metas):
        """``forward`` on the channels-last twins ``[H, W, C]`` of the current and previous
        stereo features alone (the detectors' feature cache holds only the twin)."""
        _check_cuda(cl_c, 'cur_stereo_feats (channels-last)')
        _check_cuda(cl_p, 'prev_stereo_feats (channels-last)')
        h, w, c = cl_c.shape
        assert c == self.in_channels and tuple(cl_p.shape) == (h, w, c)
        assert cl_c.is_contiguous() and cl_p.is_contiguous()
        L = self._prepare(h, w)
        geom = geometry_from_meta(img_metas[0])
        cost, stereo, mono = self._outputs(h, w, cl_c.device)
        capi.check(L.dfm_backbone_forward_cl(
            self._handle, _ptr(cl_c), _ptr(cl_p), ctypes.byref(geom), _ptr(cost),
            _ptr(stereo), _ptr(mono), _stream()), 'dfm_backbone_forward_cl')
        return self._finish(cost, stereo, mono)

    def _finish(self, cost, stereo, mono):
        # the handle keeps a channels-last copy of stereo_feat until the next forward;
        # FrustumToVoxel reads it instead of transposing `stereo` again
        self._generation = getattr(self, '_generation', 0) + 1
        stereo._dfm_channels_last = (self, self._generation)
        return cost, stereo, mono


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


_DEPTH_LOSS_TYPES = ('ce', 'balanced_ce', 'focal', 'balanced_focal')


class _DepthLossFn(torch.autograd.Function):
    """The loss of one ``dfm_depth_loss_forward``.  Forward stores the gradient of the unweighted
    loss sum when the volume requires grad; backward scales it by loss_weight^2 / count and
    ``grad_output`` on the device."""

    @staticmethod
    def forward(ctx, vol, loss, samples, depth, fg, empty):
        g = torch.empty_like(vol) if ctx.needs_input_grad[0] else None
        out, scale = loss.forward(vol, samples, depth, fg, empty, g)
        ctx.grad = g
        ctx.save_for_backward(scale)
        return out

    @staticmethod
    def backward(ctx, go):
        scale, = ctx.saved_tensors
        g = ctx.grad * (scale * go) if ctx.grad is not None else None
        return g, None, None, None, None, None


class _DepthLoss:
    """``DepthHead.loss`` through ``dfm_depth_loss_*``: one handle per (input form, shape,
    loss config, device), kept until the key changes."""

    def __init__(self):
        self.handle, self.key = None, None

    def release(self):
        if self.handle is not None:
            capi.lib().dfm_depth_loss_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def ensure(self, key, desc, dev):
        if self.handle is None or key != self.key:
            self.release()
            hd = ctypes.c_void_p()
            with torch.cuda.device(dev):
                capi.check(capi.lib().dfm_depth_loss_create(ctypes.byref(desc), ctypes.byref(hd)),
                           'dfm_depth_loss_create')
            self.handle, self.key = hd, key
            self.pixels = desc.num_images * (desc.height * desc.factor) * \
                (desc.width * desc.factor)

    def forward(self, vol, samples, depth, fg, empty, grad):
        """Runs the handle; returns the 0-dim loss and gradient scale."""
        dev = vol.device
        loss = torch.empty((), device=dev)
        scale = torch.empty((), device=dev)
        with torch.cuda.device(dev):
            capi.check(capi.lib().dfm_depth_loss_forward(
                self.handle, _ptr(vol), _ptr(samples), _ptr(depth), _ptr(fg), _ptr(empty),
                _ptr(grad), _ptr(loss), _ptr(scale), _stream()), 'dfm_depth_loss_forward')
        return loss, scale

    def workspace(self):
        """Device bytes the handle owns."""
        b = ctypes.c_longlong(0)
        capi.check(capi.lib().dfm_depth_loss_workspace(self.handle, ctypes.byref(b)),
                   'dfm_depth_loss_workspace')
        return b.value

    def debug_tensor(self, name):
        """From the last call (tests only): 'pixel_loss' fp32 [B*N, fH, fW], the weighted
        per-pixel term (0 outside the mask); 'count' int32 [1], the masked pixels."""
        if self.handle is None:
            raise RuntimeError('dfm_depth_loss_debug_tensor: no loss call has run')
        n = 1 if name == 'count' else self.pixels
        out = torch.empty(n, device='cuda',
                          dtype=torch.int32 if name == 'count' else torch.float32)
        capi.check(capi.lib().dfm_depth_loss_debug_tensor(self.handle, name.encode(), _ptr(out),
                                                          out.numel(), _stream()),
                   f'dfm_depth_loss_debug_tensor({name})')
        return out


@HEADS.register_module()
class DepthHead(_CudaMirror):
    """Drop-in for the reference ``DepthHead`` (depth_head.py:13-212): ``forward`` and ``loss``
    on CUDA."""

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
        self._depth_loss = _DepthLoss()

    def _samples_on(self, dev):
        """The injected ``depth_samples`` as fp32 on ``dev``, copied once per tensor."""
        samples = self.depth_samples
        if (self._samples_dev is None or self._samples_dev[0] is not samples
                or self._samples_dev[1].device != dev):
            self._samples_dev = (samples, samples.detach().to(dev, torch.float32).contiguous())
        return self._samples_dev[1]

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
        sdev = self._samples_on(stereo_features.device)
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

    def loss(self, depth_preds, depth_volumes, depth_img, depth_fgmask_img=None):
        """``loss_dense_depth`` (depth_head.py:75-188) on CUDA (``dfm_depth_loss_*``): a 0-dim
        device tensor, differentiable with respect to the volume.

        ``depth_volumes`` is either a ``CostLogits`` whose ``.cost`` is DfMBackbone's
        ``[B, N, D, H, W]`` logits -- the volume is then taken to be their x-downsample_factor
        trilinear (align_corners) upsampling, read column by column under the masked pixels
        without building it, and the gradient goes to ``.cost`` -- or the dense
        ``[B*N, fD, fH, fW]`` volume the reference call site passes (its gradient is zero
        outside the masked columns).  ``depth_img`` and ``depth_fgmask_img`` (any dtype,
        non-zero = foreground) are ``[B*N, fH, fW]`` CUDA tensors.  Types ``ce``,
        ``balanced_ce``, ``focal`` and ``balanced_focal``; the others raise
        ``NotImplementedError``, a balanced type without ``depth_fgmask_img`` ``ValueError``.

        Departures from the reference, all on the device with no host synchronisation:

        * the loss is multiplied by ``loss_weight`` twice, as the reference does
          (``self.loss_weight * loss_type_weight``, both ``depth_loss['loss_weight']``);
        * with no masked pixel it is ``depth_preds.mean() * 0.0`` (NaN if ``depth_preds``
          holds one), chosen on the device, with a zero gradient for the volume.  The
          reference's empty branch computes that product but returns its accumulator, the
          Python float ``0.``, and prints ``'no gt warning'``, which needs a host round trip;
          the print is left out;
        * the normaliser is the masked-pixel count over all ``B*N`` images, not all-reduced
          (as in the reference);
        * ``depth_preds`` is only checked for shape and read in the empty case; it gets no
          gradient, as under the reference's autograd when a pixel is masked;
        * sums over pixels run in fp64 (per-pixel softmax sums in fp32, as in the reference).
        """
        t = self.depth_loss_type
        if t not in _DEPTH_LOSS_TYPES:
            raise NotImplementedError(
                f"DepthHead.loss: type '{t}' is not implemented on the CUDA path; it has ce, "
                "balanced_ce, focal and balanced_focal (the shipped KITTI configs use "
                "balanced_focal)")
        balanced = t.startswith('balanced')
        if balanced and depth_fgmask_img is None:
            raise ValueError(f"DepthHead.loss: type '{t}' needs depth_fgmask_img")
        logits = isinstance(depth_volumes, CostLogits)
        vol = depth_volumes.cost if logits else depth_volumes
        f = self.downsample_factor if logits else 1
        if vol.dim() != (5 if logits else 4):
            raise RuntimeError(f'DepthHead.loss: unexpected depth_volumes shape {tuple(vol.shape)}')
        if logits:
            d, h, w = vol.shape[2:]
            n = vol.shape[0] * vol.shape[1]
        else:
            n, d, h, w = vol.shape
        if len(self.depth_samples) != f * d:
            raise RuntimeError(f'DepthHead.loss: {len(self.depth_samples)} depth_samples for '
                               f'{f * d} depth bins')
        full = (n, f * h, f * w)
        for name, x in (('depth_preds', depth_preds), ('depth_img', depth_img),
                        ('depth_fgmask_img', depth_fgmask_img)):
            if x is not None and tuple(x.shape) != full:
                raise RuntimeError(f'DepthHead.loss: {name} is {tuple(x.shape)}, expected {full}')
        _check_cuda(vol, 'depth_volumes')
        _check_cuda(depth_img, 'depth_img')
        dev = vol.device
        samples = self._samples_on(dev)
        fg = None
        if balanced:
            if not depth_fgmask_img.is_cuda or depth_fgmask_img.device != dev:
                raise RuntimeError('DepthHead.loss: depth_fgmask_img must be on the volume\'s '
                                   'device')
            fg = (depth_fgmask_img != 0).to(torch.uint8).contiguous()
        cfg = self.depth_loss
        focal = t.endswith('focal')
        alpha, gamma = (float(cfg['alpha']), float(cfg['gamma'])) if focal else (1.0, 0.0)
        fgw, bgw = (float(cfg['fg_weight']), float(cfg['bg_weight'])) if balanced else (1.0, 1.0)
        desc = (n, d, h, w, f, int(not logits), float(self.min_depth), float(self.max_depth),
                alpha, gamma, fgw, bgw, int(balanced), float(self.loss_weight))
        self._depth_loss.ensure(desc + (str(dev),), capi.DepthLossDesc(*desc), dev)
        empty = (depth_preds.detach().mean() * 0.0).to(dev, torch.float32)
        return _DepthLossFn.apply(vol.contiguous(), self._depth_loss, samples,
                                  depth_img.contiguous(), fg, empty)


class _NeckBase(_HandleMirror):
    """Debug tensors: the raw output [Nx, Ny, Zo, C] of conv layer i of a tower, 'mono.<i>' /
    'stereo.<i>' (OutdoorImVoxelNeck's one tower is 'mono')."""
    _family = 'neck'

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
        L = self._ensure((nx, ny, nz, conv_impl), lambda: (ctypes.byref(capi.NeckDesc(
            self._c0, self._cout, num_frames, nx, ny, nz, _IMPL[conv_impl])),))
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
class FrustumToVoxel(_HandleMirror):
    """Drop-in for the reference ``FrustumToVoxel``
    (necks/feature_transformation.py:12-173): same constructor arguments and
    ``state_dict`` keys (``voxel_convs.<i>.0.conv.weight`` /
    ``voxel_convs.<i>.0.gn.{weight,bias}``); ``depth_cfg`` and ``coordinates_3d``
    are injected by the detector exactly like the reference
    (detectors/dfm.py:85-100).  Debug tensors: 'vox' ([nz, ny, nx, cv], the gathered conv
    input) and 'conv<i>' (raw output of voxel_convs[i], [nz, ny, nx, 32])."""
    _family = 'frustum'

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

    def _prepare(self, d, h, w, sh, sw, f):
        """The handle for these shapes, with the current parameters (``forward`` and
        ``HotPathPipeline``)."""
        c3d = self.coordinates_3d
        key = (d, h, w, sh, sw, f, tuple(c3d.shape), c3d.data_ptr(),
               c3d._version, float(self.depth_cfg['depth_min']),
               float(self.depth_cfg['depth_max']))

        def create_args():
            nz, ny, nx = c3d.shape[:3]
            desc = capi.FrustumDesc(
                self.num_3dconvs, self.cv_channels, self.out_channels,
                self.in_sem_channels, int(self.sem_atten_feat),
                int(self.stereo_atten_feat), int(self.cat_img_feature), d, h, w, sh,
                sw, f, nx, ny, nz, float(self.depth_cfg['depth_min']),
                float(self.depth_cfg['depth_max']), _IMPL[self.conv_impl])
            # ctypes arrays own their copies of the axes for the duration of the call
            return (ctypes.byref(desc),) + tuple((ctypes.c_float * len(a))(*a.tolist())
                                                 for a in self._separable_centres(c3d))

        return self._ensure(key, create_args)

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
        L = self._prepare(d, h, w, sh, sw, f)
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
        fr._prepare(bb.num_planes, ho, wo, sem_hw[0], sem_hw[1], f)
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
    _family = 'stereo_tail'

    def __init__(self, stereo_channels=(32, 32), in_channels=32,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), conv_impl='auto'):
        super().__init__()
        assert tuple(stereo_channels) == (32, 32) and in_channels == 32
        assert norm_cfg.get('type') == 'GN' and norm_cfg.get('num_groups', 32) == 32
        self.conv_impl = conv_impl
        self.lastconv = nn.Sequential(_ConvGN2d(32, 32), nn.Conv2d(32, 32, 1, bias=False))

    def forward(self, x):
        _check_cuda(x, 'x')
        self._forward_only(x)
        b, c, h, w = x.shape
        assert c == 32
        L = self._ensure((h, w, self.conv_impl), lambda: (h, w, _IMPL[self.conv_impl]))
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
    Patch: ``model.neck = SPPUNetNeck(**cfg.model.neck)``.  Debug tensors (channels-last): raw
    conv outputs 'conv0', 'redir0', 'conv1', 'rpn0', 'rpn1', 'lastconv'; 'pool64' .. 'pool8',
    'spp64' .. 'spp8', 'concat', 'x0', 'x1'."""
    _family = 'spp_neck'

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
        L = self._ensure((h, w, self.conv_impl), lambda: (h, w, _IMPL[self.conv_impl]))
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


@BACKBONES.register_module()
class BEVHourglass(_HandleMirror):
    """Drop-in for the reference ``BEVHourglass`` forward with GroupNorm
    (backbones/bev_hourglass.py:11-137; ``backbone_3d`` of
    configs/dfm/dfm_r34_1x8_kitti-3d-3class.py:146-150).  The SyncBN variant is the frozen
    LiDAR teacher's (config :30-36, training only) and is not mirrored.  Debug tensors: the raw
    output [H, W, C] of 'compress' and 'conv1' .. 'conv6'."""
    _family = 'bev_hourglass'

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

    def forward(self, spatial_features):
        _check_cuda(spatial_features, 'spatial_features')
        self._forward_only(spatial_features)
        b, c, ny, nx = spatial_features.shape
        assert c == self.in_channels
        L = self._ensure((ny, nx, self.conv_impl), lambda: (ctypes.byref(capi.BevDesc(
            self.in_channels, self.out_channels, ny, nx, _IMPL[self.conv_impl])),))
        x = spatial_features.contiguous()
        out = torch.empty((b, self.out_channels, ny, nx), device=x.device)
        pre = torch.empty_like(out) if self.output_prehg_feat else None
        for i in range(b):
            capi.check(L.dfm_bev_hourglass_forward(
                self._handle, _ptr(x[i]), _ptr(pre[i]) if pre is not None else None,
                _ptr(out[i]), _stream()), 'dfm_bev_hourglass_forward')
        return (pre, out) if self.output_prehg_feat else out   # bev_hourglass.py:46-50


def grid_anchors(anchor_generator, ny, nx, device):
    """Anchor table ``[ny * nx * A, 7]`` of one feature level, built with the same
    ``torch.linspace`` / ``torch.tensor`` calls as the reference generators
    (core/anchor/anchor_3d_generator.py): ``Anchor3DRangeGenerator`` spaces ``n`` centres from
    min to max; ``AlignedAnchor3DRangeGenerator`` spaces ``n + 1`` and shifts them by half a
    cell.  Row ``(y * nx + x) * A + s * n_rots + r`` for range / size ``s`` and rotation ``r``,
    as ``grid_anchors(...)[0].reshape(-1, 7)``.  Anchors are copies of those values, so the
    table is the reference's bit for bit on the same device."""
    g = dict(anchor_generator)
    kind = g.get('type', 'Anchor3DRangeGenerator')
    if kind not in ('Anchor3DRangeGenerator', 'AlignedAnchor3DRangeGenerator'):
        raise NotImplementedError(f'anchor generator {kind}')
    if g.get('custom_values') or not g.get('size_per_range', True) or \
            g.get('align_corner', False):
        raise NotImplementedError('custom_values, size_per_range=False and align_corner=True '
                                  'are not implemented')
    aligned = kind == 'AlignedAnchor3DRangeGenerator'
    ranges, sizes = g['ranges'], g.get('sizes', [[3.9, 1.6, 1.56]])
    rotations = g.get('rotations', [0, 1.5707963])
    scale = g.get('scales', [1])[0]
    if len(sizes) != len(ranges):
        assert len(ranges) == 1
        ranges = ranges * len(sizes)
    extra = 1 if aligned else 0
    per_range = []
    for rng, size in zip(ranges, sizes):
        rng = torch.tensor(rng, device=device)
        axes = []
        for lo, hi, n in ((rng[2], rng[5], 1), (rng[1], rng[4], ny), (rng[0], rng[3], nx)):
            c = torch.linspace(lo, hi, n + extra, device=device)
            if aligned:
                c += (c[1] - c[0]) / 2
            axes.append(c[:n])
        z, y, x = axes
        sz = torch.tensor(size, device=device).reshape(-1, 3) * scale       # [S, 3]
        rot = torch.tensor(rotations, device=device)
        S, R = sz.shape[0], rot.shape[0]
        t = torch.empty((ny, nx, S, R, 7), device=device)
        t[..., 0] = x.view(1, nx, 1, 1)
        t[..., 1] = y.view(ny, 1, 1, 1)
        t[..., 2] = z[0]
        t[..., 3:6] = sz.view(1, 1, S, 1, 3)
        t[..., 6] = rot.view(1, 1, 1, R)
        per_range.append(t)
    return torch.cat(per_range, dim=2).reshape(-1, 7)


class _BoxPost:
    """``get_bboxes`` of both anchor heads through ``dfm_box_post_*``: one handle and anchor
    table per (feature map size, batch, device, test_cfg), kept until the key changes."""

    def __init__(self):
        self.handle, self.key = None, None

    def release(self):
        if self.handle is not None:
            capi.lib().dfm_box_post_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def run(self, head, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg, num_classes,
            use_sigmoid, dir_offset, dir_limit_offset):
        cfg = head.test_cfg if cfg is None else cfg
        if dir_cls_preds is None or any(d is None for d in dir_cls_preds):
            raise NotImplementedError('get_bboxes needs the direction classifier '
                                      '(use_direction_classifier=True)')
        if not cfg['use_rotate_nms']:
            raise NotImplementedError('use_rotate_nms=False (axis-aligned BEV NMS)')
        if len(cls_scores) != 1 or len(bbox_preds) != 1 or len(dir_cls_preds) != 1:
            raise NotImplementedError('get_bboxes takes one feature level')
        for meta in input_metas:
            bt = meta.get('box_type_3d')
            if bt is not None and getattr(bt, '__name__', '') != 'LiDARInstance3DBoxes':
                raise NotImplementedError('NMS on the BEV of LiDARInstance3DBoxes only, got '
                                          f'{bt!r}')
        B = len(input_metas)
        cls, box, dirc = (t[:B].detach().contiguous() for t in
                          (cls_scores[0], bbox_preds[0], dir_cls_preds[0]))
        for name, t in (('cls_score', cls), ('bbox_pred', box), ('dir_cls_pred', dirc)):
            _check_cuda(t, name)
        ny, nx = cls.shape[-2:]
        A, ncol = head.num_anchors, num_classes + (0 if use_sigmoid else 1)
        if cls.shape != (B, A * ncol, ny, nx) or box.shape != (B, A * 7, ny, nx) or \
                dirc.shape != (B, A * 2, ny, nx):
            raise RuntimeError(f'get_bboxes: unexpected head output shapes {tuple(cls.shape)}, '
                               f'{tuple(box.shape)}, {tuple(dirc.shape)}')
        max_num = int(cfg['max_num'])
        desc_args = (num_classes, A, ny, nx, B, int(use_sigmoid), int(cfg.get('nms_pre', -1)),
                     max_num, float(cfg.get('score_thr', 0)), float(cfg['nms_thr']),
                     float(dir_offset), float(dir_limit_offset))
        key = desc_args + (str(cls.device),)
        L = capi.lib()
        if self.handle is None or key != self.key:
            self.release()
            with torch.cuda.device(cls.device):
                anchors = grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, cls.device)
            anchors = anchors.cpu().contiguous()
            if anchors.shape[0] != ny * nx * A:
                raise RuntimeError(f'anchor generator gives {anchors.shape[0] // (ny * nx)} '
                                   f'anchors per cell, the head has {A}')
            hd = ctypes.c_void_p()
            capi.check(L.dfm_box_post_create(ctypes.byref(capi.BoxPostDesc(*desc_args)),
                                             _ptr(anchors), ctypes.byref(hd)),
                       'dfm_box_post_create')
            self.handle, self.key = hd, key
            n, nms_pre = ny * nx * A, desc_args[6]
            self.batch, self.k = B, nms_pre if 0 < nms_pre < n else n
        dev = cls.device
        boxes = torch.empty((B, max_num, 7), device=dev)
        scores = torch.empty((B, max_num), device=dev)
        labels = torch.empty((B, max_num), device=dev, dtype=torch.int32)
        count = torch.empty((B,), device=dev, dtype=torch.int32)
        with torch.cuda.device(dev):
            capi.check(L.dfm_box_post_forward(self.handle, _ptr(cls), _ptr(box), _ptr(dirc),
                                              _ptr(boxes), _ptr(scores), _ptr(labels),
                                              _ptr(count), _stream()), 'dfm_box_post_forward')
        counts = count.cpu().tolist()
        out = []
        for b, meta in enumerate(input_metas):
            k = counts[b]
            bb = boxes[b, :k]
            if meta.get('box_type_3d') is not None:
                bb = meta['box_type_3d'](bb, box_dim=7)
            out.append((bb, scores[b, :k], labels[b, :k].long()))
        return out

    def debug_tensor(self, name):
        """int32 ``[batch, K]`` stage output of the last call (tests only): 'topk_index',
        'cls<c>_candidates', 'cls<c>_keep'; -1 past each sample's count."""
        if self.handle is None:
            raise RuntimeError('dfm_box_post_debug_tensor: no get_bboxes call has run')
        out = torch.empty((self.batch, self.k), device='cuda', dtype=torch.int32)
        capi.check(capi.lib().dfm_box_post_debug_tensor(self.handle, name.encode(), _ptr(out),
                                                         out.numel(), _stream()),
                   f'dfm_box_post_debug_tensor({name})')
        return out


def _dist_reduce_mean(t):
    """``dist_reduce_mean`` (models/utils/common_utils.py): the all-reduced mean over ranks when
    ``torch.distributed`` is initialised, ``t`` itself otherwise."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        t = t / dist.get_world_size()   # a new tensor: the caller's count stays as it was
        dist.all_reduce(t)              # sums over ranks in place
    return t


def _loss_config(head, liga):
    """The loss settings both heads read from their config, with the refusals of what the shipped
    configs never use."""
    ex = head.extra_cfg
    get = (lambda k, d: ex.get(k, d)) if liga else (lambda k, d: getattr(head, k, d))
    lc, lb, ld, li = (ex.get(k) for k in ('loss_cls', 'loss_bbox', 'loss_dir', 'loss_iou'))
    if lc is None or lc.get('type') != 'FocalLoss' or not lc.get('use_sigmoid', True):
        raise NotImplementedError('loss: loss_cls must be a sigmoid FocalLoss (sampling samplers '
                                  'are not implemented)')
    if lb is None or lb.get('type') != 'SmoothL1Loss' or \
            lb.get('reduction', 'mean') != 'mean':
        raise NotImplementedError('loss: loss_bbox must be SmoothL1Loss with mean reduction')
    if not head.use_direction_classifier or ld is None or \
            ld.get('type') != 'CrossEntropyLoss' or ld.get('use_sigmoid', False):
        raise NotImplementedError('loss: needs the direction classifier with a softmax '
                                  'CrossEntropyLoss')
    if li is not None and (not liga or li.get('type') != 'IOU3DLoss'):
        raise NotImplementedError('loss: loss_iou must be LIGAAnchor3DHead\'s IOU3DLoss')
    if get('assigner_per_size', False):
        raise NotImplementedError('loss: assigner_per_size is not implemented')
    cfg = head.train_cfg or {}
    if cfg.get('code_weight'):
        raise NotImplementedError('loss: train_cfg.code_weight is not implemented')
    assigners = cfg.get('assigner')
    g = dict(ex['anchor_generator'])
    num_sizes = len(np.asarray(g.get('sizes', [[3.9, 1.6, 1.56]])).reshape(-1, 3))
    if not isinstance(assigners, (list, tuple)) or len(assigners) != num_sizes:
        raise NotImplementedError('loss: train_cfg.assigner must list one MaxIoUAssigner per '
                                  'anchor size')
    thr = []
    for a in assigners:
        if a.get('type') != 'MaxIoUAssigner' or \
                a.get('iou_calculator', {}).get('type') != 'BboxOverlapsNearest3D' or \
                a.get('iou_calculator', {}).get('coordinate', 'lidar') != 'lidar' or \
                a.get('ignore_iof_thr', -1) > 0 or not a.get('match_low_quality', True) or \
                not a.get('gt_max_assign_all', True) or \
                not isinstance(a.get('neg_iou_thr'), (int, float)):
            raise NotImplementedError(f'loss: assigner {a} is not implemented')
        thr.append((float(a['pos_iou_thr']), float(a['neg_iou_thr']),
                    float(a.get('min_pos_iou', 0.0))))
    C = head.num_classes
    return dict(
        num_classes=C, num_sizes=num_sizes,
        num_rots=len(g.get('rotations', [0, 1.5707963])),
        assign_per_class=bool(get('assign_per_class', False)),
        diff_rad_by_sin=bool(get('diff_rad_by_sin', True)), with_iou=li is not None, liga=liga,
        thr=thr, pos_weight=float(cfg.get('pos_weight', -1)),
        gamma=float(lc.get('gamma', 2.0)), alpha=float(lc.get('alpha', 0.25)),
        beta=float(lb.get('beta', 1.0)),
        loss_weight=[float(lc.get('loss_weight', 1.0)), float(lb.get('loss_weight', 1.0)),
                     float(ld.get('loss_weight', 1.0)),
                     float(li.get('loss_weight', 1.0)) if li is not None else 0.0],
        dir_offset=float(get('dir_offset', -np.pi / 2)),
        dir_limit_offset=float(get('dir_limit_offset', 0)),
        normalizer_clamp_value=float(getattr(head, 'normalizer_clamp_value', 0)),
        reduce_avg_factor=bool(getattr(head, 'reduce_avg_factor', False)) and liga)


class _AnchorLossFn(torch.autograd.Function):
    """The four loss values of one ``dfm_anchor_loss_forward`` / ``_finish``.  Forward stores the
    gradients of the loss sums of the inputs that require grad; backward scales each by its
    loss's normaliser, weight and ``grad_output``."""

    @staticmethod
    def forward(ctx, cls, box, dirc, loss):
        need = ctx.needs_input_grad
        g_cls = torch.empty_like(cls) if need[0] else None
        g_box = torch.empty_like(box) if need[1] else None
        g_dir = torch.empty_like(dirc) if need[2] else None
        g_iou = torch.empty_like(box) if need[1] and loss.cfg['with_iou'] else None
        scales = loss.forward(cls, box, dirc, g_cls, g_box, g_dir, g_iou)
        ctx.grads = (g_cls, g_box, g_dir, g_iou)
        ctx.save_for_backward(scales)
        return loss.losses

    @staticmethod
    def backward(ctx, g):
        scales, = ctx.saved_tensors
        s = scales * g
        g_cls, g_box, g_dir, g_iou = ctx.grads
        gb = g_box * s[1] if g_box is not None else None
        if g_iou is not None:
            gb = gb + g_iou * s[3]
        return (g_cls * s[0] if g_cls is not None else None, gb,
                g_dir * s[2] if g_dir is not None else None, None)


class _AnchorLoss:
    """``loss`` of both anchor heads through ``dfm_anchor_loss_*``: one handle and anchor table per
    (feature map size, batch, device, loss config), kept until the key changes."""

    def __init__(self):
        self.handle, self.key = None, None

    def release(self):
        if self.handle is not None:
            capi.lib().dfm_anchor_loss_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def run(self, head, liga, cls_scores, bbox_preds, dir_cls_preds, gt_bboxes, gt_labels,
            input_metas, gt_bboxes_ignore):
        cfg = _loss_config(head, liga)
        if gt_bboxes_ignore is not None and any(g is not None and len(g) for g in
                                                gt_bboxes_ignore):
            raise NotImplementedError('loss: gt_bboxes_ignore is not implemented')
        if len(cls_scores) != 1 or len(bbox_preds) != 1 or len(dir_cls_preds) != 1:
            raise NotImplementedError('loss takes one feature level')
        B = len(input_metas)
        if len(gt_bboxes) != B or len(gt_labels) != B:
            raise RuntimeError(f'loss: {B} input_metas, {len(gt_bboxes)} gt_bboxes and '
                               f'{len(gt_labels)} gt_labels')
        cls, box, dirc = cls_scores[0], bbox_preds[0], dir_cls_preds[0]
        for name, t in (('cls_score', cls), ('bbox_pred', box), ('dir_cls_pred', dirc)):
            _check_cuda(t, name)
        dev = cls.device
        ny, nx = cls.shape[-2:]
        A, C = head.num_anchors, cfg['num_classes']
        if A != cfg['num_sizes'] * cfg['num_rots'] or cls.shape != (B, A * C, ny, nx) or \
                box.shape != (B, A * 7, ny, nx) or dirc.shape != (B, A * 2, ny, nx):
            raise RuntimeError(f'loss: unexpected head output shapes {tuple(cls.shape)}, '
                               f'{tuple(box.shape)}, {tuple(dirc.shape)}')
        boxes, labels, off = [], [], [0]
        for gb, gl in zip(gt_bboxes, gt_labels):
            gb = gb.tensor if hasattr(gb, 'tensor') else gb
            if gb.dim() != 2 or gb.shape[1] != 7:
                raise NotImplementedError(f'loss: GT boxes must be [M, 7], got '
                                          f'{tuple(gb.shape)}')
            if gl.shape != (gb.shape[0],):
                raise RuntimeError('loss: every sample needs one label per GT box')
            # labels still on the host are checked here; on the device the kernels flag them
            # and every loss comes out NaN (no host synchronisation on the CUDA path)
            if not gl.is_cuda and gl.numel() and (int(gl.min()) < 0 or int(gl.max()) >= C):
                raise ValueError(f'loss: GT labels must lie in 0..{C - 1}')
            boxes.append(gb.to(dev, torch.float32))
            labels.append(gl.to(dev, torch.int32))
            off.append(off[-1] + gb.shape[0])
        self.gt = torch.cat(boxes).contiguous()
        self.gt_labels = torch.cat(labels).contiguous()
        self.h_off = (ctypes.c_int * (B + 1))(*off)
        self.d_off = torch.tensor(off, dtype=torch.int32).to(dev, non_blocking=True)
        t = cfg['thr'] + [(0.0, 0.0, 0.0)] * (8 - len(cfg['thr']))
        desc_args = (C, cfg['num_sizes'], cfg['num_rots'], ny, nx, B,
                     int(cfg['assign_per_class']), int(cfg['diff_rad_by_sin']), 1,
                     int(cfg['with_iou']), int(liga),
                     (ctypes.c_float * 8)(*[x[0] for x in t]),
                     (ctypes.c_float * 8)(*[x[1] for x in t]),
                     (ctypes.c_float * 8)(*[x[2] for x in t]),
                     cfg['pos_weight'], cfg['gamma'], cfg['alpha'], cfg['beta'],
                     (ctypes.c_float * 4)(*cfg['loss_weight']), cfg['dir_offset'],
                     cfg['dir_limit_offset'], cfg['normalizer_clamp_value'])
        key = (repr(sorted((k, repr(v)) for k, v in cfg.items())), ny, nx, B, str(dev))
        L = capi.lib()
        if self.handle is None or key != self.key:
            self.release()
            with torch.cuda.device(dev):
                anchors = grid_anchors(head.extra_cfg['anchor_generator'], ny, nx, dev)
            self.anchors = anchors
            anchors = anchors.cpu().contiguous()
            hd = ctypes.c_void_p()
            with torch.cuda.device(dev):
                capi.check(L.dfm_anchor_loss_create(ctypes.byref(capi.AnchorLossDesc(*desc_args)),
                                                    _ptr(anchors), ctypes.byref(hd)),
                           'dfm_anchor_loss_create')
            self.handle, self.key, self.batch, self.n = hd, key, B, ny * nx * A
        self.cfg = cfg
        losses = _AnchorLossFn.apply(cls.contiguous(), box.contiguous(), dirc.contiguous(), self)
        out = dict(loss_cls=[losses[0]], loss_bbox=[losses[1]], loss_dir=[losses[2]])
        if cfg['with_iou']:
            out['loss_iou'] = [losses[3]]
        return out

    def forward(self, cls, box, dirc, g_cls, g_box, g_dir, g_iou):
        """Runs the handle; sets ``self.losses`` [4] and returns the gradient scales [4]."""
        L = capi.lib()
        dev = cls.device
        norm = torch.empty(1, device=dev)
        with torch.cuda.device(dev):
            capi.check(L.dfm_anchor_loss_forward(
                self.handle, _ptr(cls), _ptr(box), _ptr(dirc), _ptr(self.gt),
                _ptr(self.gt_labels), _ptr(self.d_off), ctypes.cast(self.h_off, ctypes.c_void_p),
                _ptr(g_cls), _ptr(g_box), _ptr(g_dir), _ptr(g_iou), _ptr(norm), _stream()),
                'dfm_anchor_loss_forward')
            avg = _dist_reduce_mean(norm) if self.cfg['reduce_avg_factor'] else norm
            self.losses = torch.empty(4, device=dev)
            scales = torch.empty(4, device=dev)
            capi.check(L.dfm_anchor_loss_finish(self.handle, _ptr(avg), _ptr(self.losses),
                                                _ptr(scales), _stream()),
                       'dfm_anchor_loss_finish')
        return scales

    def debug_tensor(self, name):
        """Per-anchor target of the last call (tests only): 'assigned_gt', 'labels',
        'dir_targets' int32 [batch, N]; 'label_weights' fp32 [batch, N]; 'bbox_targets' fp32
        [batch, N, 7]."""
        if self.handle is None:
            raise RuntimeError('dfm_anchor_loss_debug_tensor: no loss call has run')
        shape = (self.batch, self.n) + ((7,) if name == 'bbox_targets' else ())
        dt = torch.float32 if name in ('label_weights', 'bbox_targets') else torch.int32
        out = torch.empty(shape, device='cuda', dtype=dt)
        capi.check(capi.lib().dfm_anchor_loss_debug_tensor(self.handle, name.encode(), _ptr(out),
                                                           out.numel(), _stream()),
                   f'dfm_anchor_loss_debug_tensor({name})')
        return out


_LOSS_DOC = """Training loss (``anchor3d_head.py:328-406`` with ``loss_single``{liga}) on CUDA
        (``dfm_anchor_loss_*``): ``dict(loss_cls=[t], loss_bbox=[t], loss_dir=[t]{iou})`` of 0-dim
        device tensors, differentiable with respect to the three head outputs.  ``gt_bboxes``:
        per sample ``[M, 7]`` LiDAR boxes (tensors or objects with ``.tensor``); ``gt_labels``:
        ``[M]`` ints in ``0..num_classes-1`` (host labels outside it raise ``ValueError``,
        device labels make every loss NaN).  Reads ``train_cfg`` as the reference does; one feature level, sigmoid
        FocalLoss, one MaxIoUAssigner per anchor size; refuses ``gt_bboxes_ignore`` and
        ``code_weight``.  No host synchronisation."""


@HEADS.register_module()
class LIGAAnchor3DHead(_HandleMirror):
    """Forward of the reference ``LIGAAnchor3DHead`` (dense_heads/liga_anchor3d_head.py:
    12-128): ``forward(feats) -> ([cls_score], [bbox_pred], [dir_cls_preds])``, and the
    inherited ``get_bboxes`` (anchors, decode, rotated BEV NMS) and ``loss`` (target assignment,
    the four losses and their gradients) on CUDA; the constructor keeps the reference's
    arguments so the config block builds unchanged.  Debug tensors: the raw output [ny, nx, C] of
    'cls<i>' / 'reg<i>' and of the output convs 'cls_out' (cls + dir channels) / 'reg_out', at
    their widths padded to 32."""
    _family = 'anchor_head'

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
        nd = self.num_anchors * 2 if self.use_direction_classifier else 0
        L = self._ensure((ny, nx, self.conv_impl), lambda: (ctypes.byref(capi.AnchorHeadDesc(
            self.in_channels, self.feat_channels, self.num_convs, self.cls_out_channels,
            self.num_anchors * self.box_code_size, nd, ny, nx, _IMPL[self.conv_impl])),))
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

    def get_bboxes(self, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg=None,
                   rescale=False):
        """Anchor3DHead.get_bboxes (anchor3d_head.py:407-547), which LIGAAnchor3DHead inherits:
        ``[(boxes [K, 7], scores [K], labels [K] int64)]`` per sample, on CUDA
        (``dfm_box_post_*``).  Reads ``test_cfg`` (or ``cfg``) as the reference does; sigmoid
        scores only, one feature level, rotated NMS only."""
        loss_cls = self.extra_cfg.get('loss_cls', dict(use_sigmoid=True))
        if not loss_cls.get('use_sigmoid', False):
            raise NotImplementedError('LIGAAnchor3DHead.get_bboxes: softmax scores')
        if not hasattr(self, '_box_post'):
            self._box_post = _BoxPost()
        return self._box_post.run(self, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg,
                                  self.num_classes, True,
                                  self.extra_cfg.get('dir_offset', -np.pi / 2),
                                  self.extra_cfg.get('dir_limit_offset', 0))

    def loss(self, cls_scores, bbox_preds, dir_cls_preds, gt_bboxes, gt_labels, input_metas,
             gt_bboxes_ignore=None):
        if not hasattr(self, '_anchor_loss'):
            self._anchor_loss = _AnchorLoss()
        return self._anchor_loss.run(self, True, cls_scores, bbox_preds, dir_cls_preds, gt_bboxes,
                                     gt_labels, input_metas, gt_bboxes_ignore)

    loss.__doc__ = _LOSS_DOC.format(
        liga=' of liga_anchor3d_head.py:130-226', iou=', loss_iou=[t] with loss_iou') + \
        """

        ``avg_factor`` is the all-reduced mean of ``num_total_samples`` under
        ``torch.distributed`` (``reduce_avg_factor``).  Two departures from the reference's
        ``loss_iou``: with no positive it is 0 with a zero gradient (the reference's
        ``iou3d_loss`` asserts), and each positive is decoded against its own anchor (for
        batch > 1 the reference indexes image 0's anchors with batch-wide indices and fails).
        Where a decoded target value is NaN (degenerate GT) the prediction's value stands in, as
        in ``iou3d_loss``, but the gradient does not also flow through the substituted value."""


@HEADS.register_module()
class Anchor3DHead(_HandleMirror):
    """Forward of the reference ``Anchor3DHead`` (dense_heads/anchor3d_head.py:15-185), the
    ``bbox_head_3d`` of both MultiViewDfM (Waymo) configs: ``forward(feats) -> ([cls_score],
    [bbox_pred], [dir_cls_preds or None])``.  The three 1x1 convs run as one tensor-core GEMM
    that reads the BEV map once (``csrc/head1x1_tc.cuh``); ``get_bboxes`` (anchors, decode,
    rotated BEV NMS) and ``loss`` (target assignment, losses and their gradients) run on CUDA
    too; the constructor keeps the reference's arguments so the config block builds unchanged,
    and the ``state_dict`` (``conv_cls`` / ``conv_reg`` / ``conv_dir_cls``) is the reference's."""
    _family = 'anchor3d_head'

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
        nd = self.num_anchors * 2 if self.use_direction_classifier else 0
        nr = self.num_anchors * self.box_code_size
        L = self._ensure((ny, nx, self.conv_impl), lambda: (ctypes.byref(capi.Anchor3DHeadDesc(
            self.feat_channels, self.cls_out_channels, nr, nd, ny, nx, _IMPL[self.conv_impl])),))
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

    def get_bboxes(self, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg=None,
                   rescale=False):
        """Reference ``get_bboxes`` (anchor3d_head.py:407-547): ``[(boxes [K, 7], scores [K],
        labels [K] int64)]`` per sample, on CUDA (``dfm_box_post_*``).  Reads ``test_cfg`` (or
        ``cfg``) as the reference does; one feature level, rotated NMS only."""
        if not hasattr(self, '_box_post'):
            self._box_post = _BoxPost()
        fg = self.num_classes if self.use_sigmoid_cls else self.num_classes - 1
        return self._box_post.run(self, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg,
                                  fg, self.use_sigmoid_cls, self.dir_offset,
                                  self.dir_limit_offset)

    def loss(self, cls_scores, bbox_preds, dir_cls_preds, gt_bboxes, gt_labels, input_metas,
             gt_bboxes_ignore=None):
        if not hasattr(self, '_anchor_loss'):
            self._anchor_loss = _AnchorLoss()
        return self._anchor_loss.run(self, False, cls_scores, bbox_preds, dir_cls_preds,
                                     gt_bboxes, gt_labels, input_metas, gt_bboxes_ignore)

    loss.__doc__ = _LOSS_DOC.format(liga='', iou='')


def _atss_loss_config(head):
    """The settings ``LIGAATSSHead.loss`` reads from its config, with the refusals of what no
    shipped config uses."""
    g, coder, cfg = head.anchor_generator, head.bbox_coder, head.train_cfg or {}
    asg = dict(cfg.get('assigner') or {})
    lc, lb, lz = head.loss_cls_cfg, head.loss_bbox_cfg, head.loss_centerness_cfg
    if head.reg_class_agnostic:
        raise NotImplementedError('LIGAATSSHead.loss: reg_class_agnostic=True')
    if head.num_extra_reg_channel or head.seperate_extra_reg_branch:
        raise NotImplementedError('LIGAATSSHead.loss: extra regression channels')
    if head.reg_avg_factor != 'default':
        raise NotImplementedError(f'LIGAATSSHead.loss: reg_avg_factor={head.reg_avg_factor!r}')
    if head.num_anchors != 1 or g.get('center_offset', 0.0) != 0.0 or 'scales' in g or \
            g.get('type', 'AnchorGenerator') != 'AnchorGenerator':
        raise NotImplementedError('LIGAATSSHead.loss: one anchor per location, from '
                                  'octave_base_scale, centre offset 0')
    strides = list(g['strides'])
    if not all(isinstance(s, int) and s > 0 for s in strides) or len(strides) > 8:
        raise NotImplementedError('LIGAATSSHead.loss: up to 8 levels of integer strides')
    if lc.get('type') != 'FocalLoss' or not lc.get('use_sigmoid', True) or \
            lb.get('type') != 'GIoULoss' or lz.get('type') != 'CrossEntropyLoss' or \
            not lz.get('use_sigmoid', False):
        raise NotImplementedError('LIGAATSSHead.loss: sigmoid FocalLoss, GIoULoss and sigmoid '
                                  'CrossEntropyLoss only')
    if any(lo.get('reduction', 'mean') != 'mean' for lo in (lc, lb, lz)) or \
            lz.get('class_weight') is not None or lc.get('activated', False):
        raise NotImplementedError('LIGAATSSHead.loss: mean reduction without class weights')
    if asg.get('type') != 'ATSS3DCenterAssigner' or asg.get('thresh_mode', 'meanstd') != 'meanstd' \
            or not asg.get('append_3d_centers', True) or \
            not cfg.get('append_3d_centers', True) or asg.get('ignore_iof_thr', -1) > 0:
        raise NotImplementedError('LIGAATSSHead.loss: ATSS3DCenterAssigner with '
                                  "thresh_mode='meanstd' and append_3d_centers=True only")
    if asg.get('topk') != 9 or cfg.get('allowed_border', -1) >= 0 or cfg.get('pos_weight', -1) > 0:
        raise NotImplementedError('LIGAATSSHead.loss: topk=9, allowed_border=-1 and pos_weight=-1 '
                                  'only')
    means = coder.get('target_means', [0.0] * 4)
    stds = [float(x) for x in coder.get('target_stds', [1.0] * 4)]
    if coder.get('type', 'DeltaXYWHBBoxCoder') != 'DeltaXYWHBBoxCoder' or any(means) or \
            stds[0] != stds[1] or stds[2] != stds[3] or coder.get('add_ctr_clamp', False):
        raise NotImplementedError('LIGAATSSHead.loss: DeltaXYWHBBoxCoder with means 0 and equal '
                                  'x / y and w / h stds')
    return dict(num_classes=head.num_classes, strides=strides,
                octave_base_scale=float(g['octave_base_scale']), target_stds=stds,
                wh_ratio_clip=16 / 1000, giou_eps=float(lb.get('eps', 1e-6)),
                gamma=float(lc.get('gamma', 2.0)), alpha=float(lc.get('alpha', 0.25)),
                loss_weight=[float(lc.get('loss_weight', 1.0)), float(lb.get('loss_weight', 1.0)),
                             float(lz.get('loss_weight', 1.0))])


def _ptr_table(ts):
    """A host array of device pointers (NULL for None) as a ``void *``."""
    arr = (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])
    return arr, ctypes.cast(arr, ctypes.c_void_p)


class _ATSSLossFn(torch.autograd.Function):
    """The 3 x L loss values of one ``dfm_atss_loss_forward`` / ``_finish``.  Forward stores the
    gradients of the per-level loss sums of the outputs that require grad; backward scales each
    by its loss's normaliser, weight and ``grad_output``."""

    @staticmethod
    def forward(ctx, loss, *outs):
        grads = [torch.empty_like(o) if ctx.needs_input_grad[1 + i] else None
                 for i, o in enumerate(outs)]
        scales = loss.forward(outs, grads)
        ctx.grads = grads
        ctx.save_for_backward(scales)
        return loss.losses

    @staticmethod
    def backward(ctx, g):
        scales, = ctx.saved_tensors
        s = scales * g
        return (None,) + tuple(gr * s[i] if gr is not None else None
                               for i, gr in enumerate(ctx.grads))


class _ATSSLoss:
    """``LIGAATSSHead.loss`` through ``dfm_atss_loss_*``: one handle per (feature sizes, batch,
    device, loss config), kept until the key changes."""

    def __init__(self):
        self.handle, self.key = None, None

    def release(self):
        if self.handle is not None:
            capi.lib().dfm_atss_loss_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def run(self, head, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas,
            gt_bboxes_ignore):
        cfg = _atss_loss_config(head)
        if gt_bboxes_ignore is not None and any(g is not None and len(g) for g in
                                                gt_bboxes_ignore):
            raise NotImplementedError('LIGAATSSHead.loss: gt_bboxes_ignore is not implemented')
        L, C, B = len(cfg['strides']), cfg['num_classes'], len(img_metas)
        if not (len(cls_scores) == len(bbox_preds) == len(centernesses) == L):
            raise RuntimeError(f'LIGAATSSHead.loss: {L} levels expected, got {len(cls_scores)}, '
                               f'{len(bbox_preds)}, {len(centernesses)}')
        if len(gt_bboxes) != B or len(gt_labels) != B:
            raise RuntimeError(f'LIGAATSSHead.loss: {B} img_metas, {len(gt_bboxes)} gt_bboxes and '
                               f'{len(gt_labels)} gt_labels')
        feat = []
        for lv, (c, b, z) in enumerate(zip(cls_scores, bbox_preds, centernesses)):
            for name, t in (('cls_score', c), ('bbox_pred', b), ('centerness', z)):
                _check_cuda(t, f'{name}[{lv}]')
            h, w = c.shape[-2:]
            if c.shape != (B, C, h, w) or b.shape != (B, 4 * C, h, w) or \
                    z.shape != (B, 1, h, w) or c.device != cls_scores[0].device:
                raise RuntimeError(f'LIGAATSSHead.loss: unexpected head output shapes at level '
                                   f'{lv}: {tuple(c.shape)}, {tuple(b.shape)}, {tuple(z.shape)}')
            feat.append((int(h), int(w)))
        dev = cls_scores[0].device
        boxes, labels, off = [], [], [0]
        for gb, gl in zip(gt_bboxes, gt_labels):
            if gb.dim() != 2 or gb.shape[1] != 6:
                raise RuntimeError(f'LIGAATSSHead.loss: GT must be [M, 6] (2-D box and projected '
                                   f'3-D centre), got {tuple(gb.shape)}')
            if gl.shape != (gb.shape[0],):
                raise RuntimeError('LIGAATSSHead.loss: every image needs one label per GT box')
            # labels still on the host are checked here; on the device the kernels flag them
            # and every loss comes out NaN (no host synchronisation on the CUDA path)
            if not gl.is_cuda and gl.numel() and (int(gl.min()) < 0 or int(gl.max()) >= C):
                raise ValueError(f'LIGAATSSHead.loss: GT labels must lie in 0..{C - 1}')
            boxes.append(gb.to(dev, torch.float32))
            labels.append(gl.to(dev, torch.int32))
            off.append(off[-1] + gb.shape[0])
        self.gt = torch.cat(boxes).contiguous()
        self.gt_labels = torch.cat(labels).contiguous()
        self.h_off = (ctypes.c_int * (B + 1))(*off)
        self.d_off = torch.tensor(off, dtype=torch.int32).to(dev, non_blocking=True)
        pads = [int(v) for m in img_metas for v in m['pad_shape'][:2]]
        self.h_pad = (ctypes.c_int * (2 * B))(*pads)
        key = (repr(sorted((k, repr(v)) for k, v in cfg.items())), tuple(feat), B, str(dev))
        if self.handle is None or key != self.key:
            self.release()
            z8 = lambda v: (ctypes.c_int * 8)(*v)  # noqa: E731
            desc = capi.AtssLossDesc(
                C, L, z8(cfg['strides']), z8([f[0] for f in feat]), z8([f[1] for f in feat]), B,
                9, cfg['octave_base_scale'], (ctypes.c_float * 4)(*cfg['target_stds']),
                cfg['wh_ratio_clip'], cfg['giou_eps'], cfg['gamma'], cfg['alpha'],
                (ctypes.c_float * 3)(*cfg['loss_weight']))
            hd = ctypes.c_void_p()
            with torch.cuda.device(dev):
                capi.check(capi.lib().dfm_atss_loss_create(ctypes.byref(desc), ctypes.byref(hd)),
                           'dfm_atss_loss_create')
            self.handle, self.key, self.batch = hd, key, B
            self.n = sum(h * w for h, w in feat)
        self.levels = L
        outs = [t.contiguous() for t in (*cls_scores, *bbox_preds, *centernesses)]
        losses = _ATSSLossFn.apply(self, *outs)
        return dict(loss_cls=[losses[i] for i in range(L)],
                    loss_bbox=[losses[L + i] for i in range(L)],
                    loss_centerness=[losses[2 * L + i] for i in range(L)])

    def forward(self, outs, grads):
        """Runs the handle; sets ``self.losses`` [3 L] and returns the gradient scales [3 L]."""
        L = self.levels
        lib = capi.lib()
        dev = outs[0].device
        tabs = [_ptr_table(outs[k * L:(k + 1) * L]) for k in range(3)]
        gtabs = [_ptr_table(grads[k * L:(k + 1) * L])
                 if any(g is not None for g in grads[k * L:(k + 1) * L]) else (None, None)
                 for k in range(3)]
        norm = torch.empty(2, device=dev)
        with torch.cuda.device(dev):
            capi.check(lib.dfm_atss_loss_forward(
                self.handle, tabs[0][1], tabs[1][1], tabs[2][1], _ptr(self.gt),
                _ptr(self.gt_labels), _ptr(self.d_off), ctypes.cast(self.h_off, ctypes.c_void_p),
                ctypes.cast(self.h_pad, ctypes.c_void_p), gtabs[0][1], gtabs[1][1], gtabs[2][1],
                _ptr(norm), _stream()), 'dfm_atss_loss_forward')
            # num_total_pos and the centerness sum, all-reduced in one call
            avg = _dist_reduce_mean(norm)
            self.losses = torch.empty(3 * L, device=dev)
            scales = torch.empty(3 * L, device=dev)
            capi.check(lib.dfm_atss_loss_finish(self.handle, _ptr(avg), _ptr(self.losses),
                                                _ptr(scales), _stream()),
                       'dfm_atss_loss_finish')
        return scales

    def debug_tensor(self, name):
        """Per-anchor target of the last call (tests only): 'assigned_gt', 'labels' int32
        [batch, N]; 'label_weights', 'centerness_targets' fp32 [batch, N]; 'bbox_targets' fp32
        [batch, N, 4]; 'thresholds' fp32 [G]."""
        if self.handle is None:
            raise RuntimeError('dfm_atss_loss_debug_tensor: no loss call has run')
        shape = {'bbox_targets': (self.batch, self.n, 4),
                 'thresholds': (self.gt.shape[0],)}.get(name, (self.batch, self.n))
        dt = torch.int32 if name in ('assigned_gt', 'labels') else torch.float32
        out = torch.empty(shape, device=self.gt.device, dtype=dt)
        capi.check(capi.lib().dfm_atss_loss_debug_tensor(self.handle, name.encode(), _ptr(out),
                                                         out.numel(), _stream()),
                   f'dfm_atss_loss_debug_tensor({name})')
        return out


class _Scale(nn.Module):
    """mmcv ``Scale``: a learnable scalar factor."""

    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))

    def forward(self, x):
        return x * self.scale


@HEADS.register_module()
class LIGAATSSHead(nn.Module):
    """DfM's 2-D auxiliary head (dense_heads/liga_atss_head.py, an mmdet ``ATSSHead``): the
    reference constructor and ``state_dict`` keys, a plain differentiable PyTorch ``forward``
    (the head is trained: ConvModule = 3 x 3 conv without bias, GroupNorm, ReLU; ``Scale`` and
    ``.float()`` on ``bbox_pred``), and ``loss`` on CUDA (``dfm_atss_loss_*``).  Registered in
    this package's ``HEADS`` only; ``DfM`` does not build it."""

    def __init__(self, num_classes, in_channels, stacked_convs=4, conv_cfg=None,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                 loss_centerness=dict(type='CrossEntropyLoss', use_sigmoid=True,
                                      loss_weight=1.0),
                 reg_class_agnostic=True, num_extra_reg_channel=0,
                 seperate_extra_reg_branch=False, reg_avg_factor='default', feat_channels=256,
                 anchor_generator=dict(type='AnchorGenerator', ratios=[1.0],
                                       octave_base_scale=8, scales_per_octave=1,
                                       strides=[8, 16, 32, 64, 128]),
                 bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[.0, .0, .0, .0],
                                 target_stds=[0.1, 0.1, 0.2, 0.2]),
                 loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25,
                               loss_weight=1.0),
                 loss_bbox=dict(type='GIoULoss', loss_weight=2.0), train_cfg=None,
                 test_cfg=None, init_cfg=None, **kwargs):
        super().__init__()
        assert reg_avg_factor in ('default', 'sum_centerness')
        assert conv_cfg is None and norm_cfg is not None and norm_cfg.get('type') == 'GN', \
            'only the GroupNorm ConvModule is implemented'
        self.num_classes, self.in_channels = num_classes, in_channels
        self.feat_channels, self.stacked_convs = feat_channels, stacked_convs
        self.reg_class_agnostic, self.reg_avg_factor = reg_class_agnostic, reg_avg_factor
        self.num_extra_reg_channel = num_extra_reg_channel
        self.num_reg_channel = num_extra_reg_channel + 4
        self.seperate_extra_reg_branch = seperate_extra_reg_branch and self.num_reg_channel > 4
        self.anchor_generator, self.bbox_coder = dict(anchor_generator), dict(bbox_coder)
        self.loss_cls_cfg, self.loss_bbox_cfg = dict(loss_cls), dict(loss_bbox)
        self.loss_centerness_cfg = dict(loss_centerness)
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.extra_cfg = kwargs
        g = anchor_generator
        self.num_anchors = len(g.get('ratios', [1.0])) * (
            g.get('scales_per_octave', 1) if 'octave_base_scale' in g else len(g.get('scales', [1])))
        self.cls_out_channels = num_classes      # sigmoid classification
        ng = norm_cfg.get('num_groups', 32)

        def conv_module(cin):
            m = _ConvGN2d(cin, feat_channels)
            m.gn = nn.GroupNorm(ng, feat_channels)
            return m

        # _init_layers (liga_atss_head.py:46-128)
        self.cls_convs = nn.ModuleList([conv_module(in_channels if i == 0 else feat_channels)
                                        for i in range(stacked_convs)])
        self.reg_convs = nn.ModuleList([conv_module(in_channels if i == 0 else feat_channels)
                                        for i in range(stacked_convs)])
        if self.seperate_extra_reg_branch:
            self.extra_reg_convs = nn.ModuleList(
                [conv_module(in_channels if i == 0 else feat_channels)
                 for i in range(stacked_convs)])
        A, R = self.num_anchors, self.num_reg_channel
        self.atss_cls = nn.Conv2d(feat_channels, A * num_classes, 3, padding=1)
        per = 1 if reg_class_agnostic else num_classes
        if not self.seperate_extra_reg_branch:
            self.atss_reg = nn.Conv2d(feat_channels, A * R * per, 3, padding=1)
        else:
            self.atss_reg = nn.Conv2d(feat_channels, A * 4 * per, 3, padding=1)
            self.atss_extra_reg = nn.Conv2d(feat_channels, A * (R - 4) * per, 3, padding=1)
        self.atss_centerness = nn.Conv2d(feat_channels, A, 3, padding=1)
        self.scales = nn.ModuleList([_Scale(1.0) for _ in g['strides']])
        # ATSSHead.init_weights: normal(std 0.01), classification bias at prior 0.01
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, 0.0, 0.01)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        nn.init.constant_(self.atss_cls.bias, float(-np.log((1 - 0.01) / 0.01)))

    @staticmethod
    def _tower(convs, x):
        for m in convs:
            x = torch.relu(m.gn(m.conv(x)))
        return x

    def forward(self, feats):
        """``(cls_scores, bbox_preds, centernesses)``, one entry per level."""
        outs = [self.forward_single(x, s) for x, s in zip(feats, self.scales)]
        return tuple(map(list, zip(*outs)))

    def forward_single(self, x, scale):
        if self.seperate_extra_reg_branch:
            raise NotImplementedError('LIGAATSSHead: seperate_extra_reg_branch')
        cls_feat = self._tower(self.cls_convs, x)
        reg_feat = self._tower(self.reg_convs, x)
        cls_score = self.atss_cls(cls_feat)
        bbox_pred = scale(self.atss_reg(reg_feat)).float()
        centerness = self.atss_centerness(reg_feat)
        return cls_score, bbox_pred, centerness

    def loss(self, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas,
             gt_bboxes_ignore=None):
        """``ATSSHead.loss`` with LIGA's ``loss_single`` (liga_atss_head.py:176-270) on CUDA:
        ``dict(loss_cls=[L], loss_bbox=[L], loss_centerness=[L])`` of 0-dim device tensors,
        differentiable with respect to the 3 x L head outputs (fp32 CUDA tensors).
        ``gt_bboxes``: per image ``[M, 6]``, the 2-D box then the projected 3-D centre;
        ``gt_labels``: ``[M]`` ints in ``0..num_classes-1`` (host labels outside it raise
        ``ValueError``, device labels make every loss NaN); ``img_metas``: ``pad_shape`` per
        image.  Both normalisers are all-reduced means under ``torch.distributed``.  Refuses
        ``gt_bboxes_ignore``, ``reg_class_agnostic``, extra regression channels,
        ``reg_avg_factor='sum_centerness'``, several anchors per location, other assigner modes
        and other loss types with ``NotImplementedError``.  No host synchronisation."""
        if not hasattr(self, '_atss_loss'):
            self._atss_loss = _ATSSLoss()
        return self._atss_loss.run(self, cls_scores, bbox_preds, centernesses, gt_bboxes,
                                   gt_labels, img_metas, gt_bboxes_ignore)


class _ImitationLossFn(torch.autograd.Function):
    """The per-pair losses of one ``dfm_imitation_loss_forward`` / ``_finish``.  When an input
    requires grad, forward also runs ``dfm_imitation_loss_backward`` (grad_output 1) while the
    handle's workspace still holds this call's mask; backward scales each stored gradient by its
    loss's ``grad_output``."""

    @staticmethod
    def forward(ctx, run, *tensors):
        P = len(run.pairs)
        need = ctx.needs_input_grad[1:]
        xs, ws, bs = tensors[:P], tensors[P:2 * P], tensors[2 * P:]
        gx = [torch.empty_like(x) if need[i] else None for i, x in enumerate(xs)]
        gw = [torch.empty_like(w) if need[P + i] else None for i, w in enumerate(ws)]
        gb = [torch.empty_like(b) if need[2 * P + i] else None for i, b in enumerate(bs)]
        losses, coef = run.forward(xs, ws, bs)
        if any(need):
            run.backward(coef, gx, gw, gb)
        ctx.grads = gx + gw + gb
        return losses

    @staticmethod
    def backward(ctx, go):
        P = len(ctx.grads) // 3
        return (None,) + tuple(g * go[i % P] if g is not None else None
                               for i, g in enumerate(ctx.grads))


class _ImitationLoss:
    """``DfMImitation.loss`` through ``dfm_imitation_loss_*``: one handle per (shape, batch,
    config, device), kept until the key changes."""

    def __init__(self):
        self.handle, self.key, self.anchors = None, None, None

    def release(self):
        if self.handle is not None:
            capi.lib().dfm_imitation_loss_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def anchor_xy(self, anchor_generator, ny, nx, dev):
        """The BEV cells' anchor centres ``[nx + ny]`` (x per column, then y per row): columns 0
        and 1 of ``grid_anchors`` rows ``(y * nx + x) * A``."""
        key = (ny, nx, str(dev))
        if self.anchors is None or self.anchors[0] != key:
            with torch.cuda.device(dev):
                a = grid_anchors(anchor_generator, ny, nx, dev)
            A = a.shape[0] // (ny * nx)
            xy = torch.cat((a[0:nx * A:A, 0], a[0::nx * A, 1])).contiguous()
            self.anchors = (key, xy)
        return self.anchors[1]

    def run(self, mod, xs, ts, scales, gt_bboxes_3d):
        B, ny, nx = xs[0].shape[0], xs[0].shape[-2], xs[0].shape[-1]
        dev = xs[0].device
        if len(gt_bboxes_3d) != B:
            raise RuntimeError(f'DfMImitation.loss: {B} samples, {len(gt_bboxes_3d)} gt_bboxes_3d')
        boxes, off = [], [0]
        for gb in gt_bboxes_3d:
            gb = gb.tensor if hasattr(gb, 'tensor') else gb
            if not isinstance(gb, torch.Tensor) or gb.dim() != 2 or gb.shape[1] < 7:
                raise RuntimeError('DfMImitation.loss: GT boxes must be [M, 7] per sample, got '
                                   f'{tuple(gb.shape) if isinstance(gb, torch.Tensor) else gb}')
            boxes.append(gb[:, :7].to(dev, torch.float32))
            off.append(off[-1] + gb.shape[0])
        self.gt = torch.cat(boxes).contiguous()
        self.h_off = (ctypes.c_int * (B + 1))(*off)
        self.d_off = torch.tensor(off, dtype=torch.int32).to(dev, non_blocking=True)
        self.anchor = self.anchor_xy(mod.anchor_generator, ny, nx, dev)
        self.pairs = [(x.shape[1], x.shape[2] if x.dim() == 5 else 1) for x in xs]
        lw = [float(c['loss_weight']) for c in mod.imitation_cfgs]
        P = len(self.pairs)
        desc = (B, ny, nx, P, tuple(c for c, _ in self.pairs), tuple(z for _, z in self.pairs),
                tuple(lw), float(mod.normalizer_clamp_value))
        key = desc + (str(dev),)
        if self.handle is None or key != self.key:
            self.release()
            pad = lambda v: v + (0,) * (2 - len(v))  # noqa: E731
            d = capi.ImitationLossDesc(B, ny, nx, P, (ctypes.c_int * 2)(*pad(desc[4])),
                                       (ctypes.c_int * 2)(*pad(desc[5])),
                                       (ctypes.c_float * 2)(*pad(desc[6])), desc[7])
            hd = ctypes.c_void_p()
            with torch.cuda.device(dev):
                capi.check(capi.lib().dfm_imitation_loss_create(ctypes.byref(d), ctypes.byref(hd)),
                           'dfm_imitation_loss_create')
            self.handle, self.key = hd, key
        self.ts, self.scales, self.training = ts, scales, mod.training
        ws = [c.weight for c in mod._convs()]
        bs = [c.bias for c in mod._convs()]
        losses = _ImitationLossFn.apply(self, *xs, *ws, *bs)
        return [losses[i] for i in range(P)]

    def forward(self, xs, ws, bs):
        """Runs forward, the all-reduce of the packed counts and sums, and finish; returns the
        losses [P] and the gradient coefficients [P]."""
        import torch.distributed as dist
        lib = capi.lib()
        dev = xs[0].device
        P = len(xs)
        tabs = [_ptr_table(v) for v in (xs, self.ts, ws, bs, self.scales)]
        packed = torch.empty(sum(2 + c for c, _ in self.pairs), device=dev)
        ranks = dist.is_available() and dist.is_initialized()
        world = dist.get_world_size() if ranks else 1
        with torch.cuda.device(dev):
            capi.check(lib.dfm_imitation_loss_forward(
                self.handle, tabs[0][1], tabs[1][1], tabs[2][1], tabs[3][1], tabs[4][1],
                _ptr(self.anchor), _ptr(self.gt) if self.gt.numel() else None, _ptr(self.d_off),
                ctypes.cast(self.h_off, ctypes.c_void_p), world, _ptr(packed), _stream()),
                'dfm_imitation_loss_forward')
            # every pair's count / world, count and per-channel |t| sums in one all-reduce
            if ranks:
                dist.all_reduce(packed)
            losses = torch.empty(P, device=dev)
            coef = torch.empty(P, device=dev)
            capi.check(lib.dfm_imitation_loss_finish(self.handle, _ptr(packed),
                                                     int(self.training), _ptr(losses),
                                                     _ptr(coef), _stream()),
                       'dfm_imitation_loss_finish')
        return losses, coef

    def backward(self, coef, gx, gw, gb):
        tabs = [_ptr_table(v) if any(g is not None for g in v) else (None, None)
                for v in (gx, gw, gb)]
        with torch.cuda.device(coef.device):
            capi.check(capi.lib().dfm_imitation_loss_backward(
                self.handle, _ptr(coef), None, tabs[0][1], tabs[1][1], tabs[2][1], _stream()),
                'dfm_imitation_loss_backward')

    def workspace(self):
        """Device bytes the handle owns."""
        b = ctypes.c_longlong(0)
        capi.check(capi.lib().dfm_imitation_loss_workspace(self.handle, ctypes.byref(b)),
                   'dfm_imitation_loss_workspace')
        return b.value

    def debug_tensor(self, name):
        """From the last call (tests only): 'inbox' uint8 [B, ny, nx]; 'counts' int32 [P], this
        rank's positives per pair; 'loss_sums' fp64 [P]."""
        if self.handle is None:
            raise RuntimeError('dfm_imitation_loss_debug_tensor: no loss call has run')
        B, ny, nx = self.key[:3]
        shape, dt = {'inbox': ((B, ny, nx), torch.uint8),
                     'counts': ((len(self.pairs),), torch.int32),
                     'loss_sums': ((len(self.pairs),), torch.float64)}.get(
                         name, ((0,), torch.float32))
        out = torch.empty(shape, device=self.gt.device, dtype=dt)
        capi.check(capi.lib().dfm_imitation_loss_debug_tensor(self.handle, name.encode(),
                                                              _ptr(out), out.numel(), _stream()),
                   f'dfm_imitation_loss_debug_tensor({name})')
        return out


class _NormalizeLayer(nn.Module):
    """Parameter layout of the reference's ``NormalizeLayer('cw_scale', channel)``
    (detectors/imitation_utils.py:10-94): the running per-channel scale ``[1, C]``, which
    ``DfMImitation.loss`` divides the teacher by and updates in training mode."""

    def __init__(self, channel, momentum=0.99):
        super().__init__()
        self.type, self.channel, self.momentum = 'cw_scale', channel, momentum
        self.register_buffer('scale', torch.ones(1, channel))


class DfMImitation(nn.Module):
    """DfM's LiDAR imitation loss (``DfM.imitation_loss``, detectors/dfm.py:455-539) with the
    reference's imitation layers (``_init_imitation_layers``, :213-262): ``conv_imitation`` (a
    ``ModuleList`` of 1x1 ``Conv2d`` / ``Conv3d`` with bias, or the one conv of a single config)
    and ``norm_imitation`` (per stereo feature name, the running ``cw_scale``), with the
    reference's ``state_dict`` keys.  Build it from the detector config's ``imitation_cfgs``,
    ``bbox_head_3d['anchor_generator']`` and ``normalizer_clamp_value``.  The conv layers are
    ordinary trainable parameters; the loss and its gradients run on CUDA
    (``dfm_imitation_loss_*``).  Configurations the shipped KITTI configs do not use (mode
    'full', kernel_size > 1, use_relu, layer 'none', a normalize type other than 'cw_scale', or
    channel counts other than 16 / 32 / 64) raise ``NotImplementedError``."""

    def __init__(self, imitation_cfgs, anchor_generator, normalizer_clamp_value=10):
        super().__init__()
        cfgs = list(imitation_cfgs) if isinstance(imitation_cfgs, (list, tuple)) \
            else [imitation_cfgs]
        if not 1 <= len(cfgs) <= 2:
            raise NotImplementedError('DfMImitation takes one or two imitation configs')
        for c in cfgs:
            if c.get('mode') != 'inbox':
                raise NotImplementedError(f"DfMImitation: mode {c.get('mode')!r} is not "
                                          "implemented (the shipped configs use 'inbox')")
            if c.get('layer') not in ('conv2d', 'conv3d'):
                raise NotImplementedError(f"DfMImitation: layer {c.get('layer')!r} is not "
                                          'implemented (conv2d and conv3d are)')
            if c.get('kernel_size') != 1 or c.get('use_relu'):
                raise NotImplementedError('DfMImitation: only 1x1 convs without ReLU are '
                                          'implemented')
            if c.get('normalize') != 'cw_scale':
                raise NotImplementedError(f"DfMImitation: normalize {c.get('normalize')!r} is "
                                          "not implemented (the shipped configs use 'cw_scale')")
            if c.get('channel') not in (16, 32, 64):
                raise NotImplementedError('DfMImitation: channel must be 16, 32 or 64')
        self.imitation_cfgs = cfgs
        self.anchor_generator = dict(anchor_generator)
        self.normalizer_clamp_value = normalizer_clamp_value
        convs = []
        self.norm_imitation = nn.ModuleDict()
        for c in cfgs:
            conv = nn.Conv2d if c['layer'] == 'conv2d' else nn.Conv3d
            convs.append(conv(c['channel'], c['channel'], kernel_size=1, padding=0, stride=1,
                              groups=1))
            self.norm_imitation[c['stereo_feature_layer']] = _NormalizeLayer(c['channel'])
        self.conv_imitation = nn.ModuleList(convs) if len(convs) > 1 else convs[0]
        self._loss = _ImitationLoss()

    def _convs(self):
        return list(self.conv_imitation) if len(self.imitation_cfgs) > 1 \
            else [self.conv_imitation]

    def loss(self, stereo_features, lidar_features, gt_bboxes_3d):
        """The imitation losses ``[loss per config]`` (0-dim device tensors), as
        ``losses['loss_imitation']`` holds them.  ``stereo_features`` / ``lidar_features``: dicts
        of the stereo and teacher features by the configs' ``stereo_feature_layer`` /
        ``lidar_feature_layer`` names (``spatial_features_2d`` ``[B, 64, ny, nx]``,
        ``volume_features`` ``[B, 32, nz, ny, nx]``), fp32 CUDA tensors.  ``gt_bboxes_3d``: per
        sample ``[M, 7]`` LiDAR boxes (tensors or objects with ``.tensor``).  Differentiable with
        respect to the stereo features and the conv weights and biases; the teacher and the
        scales get no gradient.  In training mode the scales are updated in place.  No host
        synchronisation.

        Departures from the reference, which runs only at B = 1 and only with a process group:
        each sample is tested against its own GT (ragged lists, any B), the normaliser counts
        the whole batch and the loss divides by B (the reference at B = 1); the counts and sums
        are all-reduced only when ``torch.distributed`` is initialised; the update's ``n > 10``
        gate is taken on the device; the anchor centres come from ``grid_anchors`` (the
        reference's ``anchors[0][:, :, :, 0, 0, :3]`` indexes a list of lists and raises);
        ``tb_dict`` is not computed."""
        xs, ts, scales = [], [], []
        ref = None
        for c in self.imitation_cfgs:
            sname, lname = c['stereo_feature_layer'], c['lidar_feature_layer']
            if sname not in stereo_features or lname not in lidar_features:
                raise RuntimeError(f'DfMImitation.loss: needs stereo {sname!r} and teacher '
                                   f'{lname!r} features')
            x, t = stereo_features[sname], lidar_features[lname]
            scale = self.norm_imitation[sname].scale
            for name, v in ((sname, x), (lname, t), (f'norm_imitation.{sname}.scale', scale)):
                _check_cuda(v, name)
            dims = 4 if c['layer'] == 'conv2d' else 5
            if x.dim() != dims or x.shape != t.shape or x.shape[1] != c['channel'] or \
                    (ref is not None and (x.shape[0], *x.shape[-2:]) != ref) or \
                    x.device != t.device or scale.device != x.device:
                raise RuntimeError(f'DfMImitation.loss: stereo {tuple(x.shape)} and teacher '
                                   f'{tuple(t.shape)} features of {sname!r} do not match each '
                                   f'other, the config or the other pair')
            ref = (x.shape[0], *x.shape[-2:])
            xs.append(x.contiguous())
            ts.append(t.detach().contiguous())
            scales.append(scale)
        for conv in self._convs():
            for v in (conv.weight, conv.bias):
                _check_cuda(v, 'conv_imitation')
                if v.device != xs[0].device:
                    raise RuntimeError('DfMImitation.loss: the layers and features are on '
                                       'different devices')
        return self._loss.run(self, xs, ts, scales, gt_bboxes_3d)

    def debug_tensor(self, name):
        return self._loss.debug_tensor(name)

    def workspace(self):
        return self._loss.workspace()


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
    Patch: ``model.neck = FPN(**cfg.model.neck)``.  Debug tensors (channels-last [B, H, W, C]):
    the merged laterals 'merged0' .. 'merged3' and the raw fpn_conv outputs before the bias
    'fpn0' .. 'fpn3'."""
    _family = 'fpn'

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

        def create_args():
            desc = capi.FpnDesc()
            desc.in_channels[:] = self.in_channels
            desc.out_channels = self.out_channels
            desc.level_h[:] = [s[0] for s in sizes]
            desc.level_w[:] = [s[1] for s in sizes]
            desc.num_images, desc.conv_impl = b, _IMPL[self.conv_impl]
            return (ctypes.byref(desc),)

        L = self._ensure((tuple(sizes), self.conv_impl), create_args, batch=b)
        xs = [x.contiguous() for x in inputs]
        arr = ctypes.c_void_p * 4
        capi.check(L.dfm_fpn_forward(self._handle, arr(*[x.data_ptr() for x in xs]),
                                     arr(*[o.data_ptr() for o in outs]), _stream()),
                   'dfm_fpn_forward')
        return outs


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
    Patch: ``model.backbone = LIGAResNet(**cfg.model.backbone)``.  Debug tensors (channels-last
    [B, h, w, C]): 'stem' (raw conv1), 'layerI.J.conv1' / 'layerI.J.conv2' /
    'layer2.0.downsample' (raw conv outputs) and the block outputs 'layerI.J'."""
    _family = 'liga_resnet'
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
        L = self._ensure((h, w, self.conv_impl), lambda: (ctypes.byref(capi.LigaResNetDesc(
            h, w, b, _IMPL[self.conv_impl])),), batch=b)
        x = img.contiguous()
        arr = ctypes.c_void_p * 4
        capi.check(L.dfm_liga_resnet_forward(self._handle, _ptr(x),
                                             arr(*[o.data_ptr() for o in outs]), _stream()),
                   'dfm_liga_resnet_forward')
        return outs


class _ModulatedDeformConv2dPack(nn.Module):
    """Parameter layout of mmcv's ``ModulatedDeformConv2dPack`` as DCNv2 builds it (3x3, no bias,
    deform_groups 1): ``weight`` and ``conv_offset`` (3x3 conv to 27 channels with a bias)."""

    def __init__(self, inplanes, planes, stride):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(planes, inplanes, 3, 3))
        self.conv_offset = nn.Conv2d(inplanes, 27, 3, stride, 1, bias=True)
        self.stride = stride


class _Bottleneck(nn.Module):
    """Parameter layout of mmdet's ``Bottleneck`` (style 'pytorch'): conv1 / bn1 / conv2 / bn2 /
    conv3 / bn3 and an optional ``downsample`` = (1x1 conv, BatchNorm)."""

    def __init__(self, inplanes, planes, stride, dcn, downsample):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _ModulatedDeformConv2dPack(planes, planes, stride) if dcn else \
            nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = nn.Sequential(
            nn.Conv2d(inplanes, planes * 4, 1, stride, bias=False),
            nn.BatchNorm2d(planes * 4)) if downsample else None
        self.stride = stride


@BACKBONES.register_module()
class ResNet(_HandleMirror):
    """mmdet's ``ResNet`` (mmdet/models/backbones/resnet.py, 2.x) in the configuration of both
    MultiViewDfM (Waymo) configs' ``backbone`` on CUDA (``csrc/resnet101_api.inc``): depth 101,
    style 'pytorch', the default strides (1, 2, 2, 2), dilations and out_indices, max-pool stem,
    and ``dcn=dict(type='DCNv2', deform_groups=1, fallback_on_stride=False)`` in layer3 / layer4
    (every conv2 there is a modulated deformable conv, the stride-2 ones included).
    ``forward(img [B, 3, H, W]) -> tuple`` of 4 NCHW maps [B, 256, H/4, W/4], [B, 512, H/8, W/8],
    [B, 1024, H/16, W/16], [B, 2048, H/32, W/32] (PyTorch's output sizes: each stride-2 step
    rounds up) for any batch size in one C call.  The ``state_dict`` is mmdet's (676 entries,
    BatchNorm running statistics and ``conv2.conv_offset`` included); BatchNorm runs in eval
    form.  ``frozen_stages``, ``norm_eval``, ``init_cfg`` / ``pretrained``, ``with_cp`` and
    ``zero_init_residual`` are accepted and ignored; any other setting (other depths, no DCN,
    other DCN placement, caffe style, deep stem, plugins, non-BN norms, ...) raises
    ``NotImplementedError``.  It is registered in the local ``BACKBONES`` only, never over
    mmdet's global ``ResNet`` (forward-only: training keeps mmdet's class).
    Patch: ``model.backbone = ResNet(**cfg.model.backbone)``.  Debug tensors (channels-last
    [B, h, w, C]): 'stem' (raw conv1), 'pool', 'layerI.J.conv1' / '.conv2' / '.conv3' /
    'layerI.0.downsample' (raw conv outputs), 'layerI.J.conv2.conv_offset' (conv_offset + bias,
    32 channels of which 27 are real), 'layerI.J.conv2.offset_mask' (the same with the sigmoid
    on channels 18..26) and the block outputs 'layerI.J'."""
    _family = 'resnet101'
    STAGE_BLOCKS = (3, 4, 23, 3)
    DCN = dict(type='DCNv2', deform_groups=1, fallback_on_stride=False)

    def __init__(self, depth, in_channels=3, stem_channels=None, base_channels=64, num_stages=4,
                 strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3),
                 style='pytorch', deep_stem=False, avg_down=False, frozen_stages=-1,
                 conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), norm_eval=True,
                 dcn=None, stage_with_dcn=(False, False, False, False), plugins=None,
                 with_cp=False, zero_init_residual=True, pretrained=None, init_cfg=None,
                 conv_impl='auto'):
        super().__init__()
        dcn_ok = isinstance(dcn, dict) and dict(dcn) == self.DCN
        checks = (
            (depth == 101, f'depth={depth}'),
            (in_channels == 3 and stem_channels in (None, 64) and base_channels == 64,
             'in_channels / stem_channels / base_channels other than 3 / 64 / 64'),
            (num_stages == 4 and tuple(strides) == (1, 2, 2, 2) and
             tuple(dilations) == (1, 1, 1, 1), f'strides={strides}, dilations={dilations}'),
            (tuple(out_indices) == (0, 1, 2, 3), f'out_indices={out_indices}'),
            (style == 'pytorch', f'style={style!r}'),
            (not deep_stem, 'deep_stem'), (not avg_down, 'avg_down'),
            (dcn_ok, f'dcn={dcn}'),
            (tuple(stage_with_dcn) == (False, False, True, True),
             f'stage_with_dcn={stage_with_dcn}'),
            (plugins is None, 'plugins'), (conv_cfg is None, 'conv_cfg'),
            (norm_cfg is not None and norm_cfg.get('type') in ('BN', 'SyncBN'),
             f'norm_cfg={norm_cfg}'))
        for ok, what in checks:
            if not ok:
                raise NotImplementedError(
                    f'ResNet: {what} is not implemented (only the Waymo backbone: depth 101, '
                    "style 'pytorch', default strides / dilations, DCNv2 (deform_groups 1, "
                    'fallback_on_stride False) in layer3 / layer4, BatchNorm)')
        self.depth, self.num_stages = depth, num_stages
        self.strides, self.dilations = tuple(strides), tuple(dilations)
        self.out_indices, self.style = tuple(out_indices), style
        self.frozen_stages, self.norm_cfg, self.norm_eval = frozen_stages, norm_cfg, norm_eval
        self.dcn, self.stage_with_dcn = dict(dcn), tuple(stage_with_dcn)
        self.with_cp, self.zero_init_residual = with_cp, zero_init_residual
        self.pretrained, self.init_cfg = pretrained, init_cfg
        self.conv_impl = conv_impl
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.res_layers = []
        inplanes = 64
        for i, n in enumerate(self.STAGE_BLOCKS):
            planes = 64 << i
            blocks = []
            for j in range(n):
                stride = self.strides[i] if j == 0 else 1
                blocks.append(_Bottleneck(inplanes, planes, stride, self.stage_with_dcn[i],
                                          j == 0))
                inplanes = planes * 4
            self.add_module(f'layer{i + 1}', nn.Sequential(*blocks))
            self.res_layers.append(f'layer{i + 1}')

    @staticmethod
    def output_sizes(h, w):
        """[(H2, W2) of the stem, (H4, W4), (H8, W8), (H16, W16), (H32, W32)]: PyTorch's
        output-size rule of every stride-2 step (ceil(n / 2))."""
        out = []
        for _ in range(5):
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            out.append((h, w))
        return out

    @staticmethod
    def check_shapes(img):
        """Raises ValueError on an input that is not [B, 3, H, W] with a non-empty image."""
        if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[1] != 3 or \
                img.shape[2] < 1 or img.shape[3] < 1:
            shape = tuple(img.shape) if isinstance(img, torch.Tensor) else type(img).__name__
            raise ValueError(f'ResNet takes an image batch [B, 3, H, W], got {shape}')

    def forward(self, img):
        self.check_shapes(img)
        _check_cuda(img, 'img')
        self._forward_only(img)
        b, _, h, w = img.shape
        sizes = self.output_sizes(h, w)[1:]
        dev = img.device
        outs = tuple(torch.empty((b, 256 << l) + sizes[l], device=dev) for l in range(4))
        if b == 0:
            return outs
        L = self._ensure((h, w, self.conv_impl), lambda: (ctypes.byref(capi.ResNet101Desc(
            h, w, b, _IMPL[self.conv_impl])),), batch=b)
        x = img.contiguous()
        arr = ctypes.c_void_p * 4
        capi.check(L.dfm_resnet101_forward(self._handle, _ptr(x),
                                           arr(*[o.data_ptr() for o in outs]), _stream()),
                   'dfm_resnet101_forward')
        return outs


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
    feats: [T*Nv, C, Hf, Wf] CUDA, or a sequence of T*Nv [C, Hf, Wf] CUDA views anywhere in
    memory (the kernel reads them through a pointer table, so cached and freshly computed views
    are lifted without a concatenation) -> [C(*T), Nx, Ny, Nz].  The returned tensor has the
    reference's shape but channels-last strides (memory [Nx, Ny, Nz, C]): that is what the
    necks' conv loaders read, so neither the lifting kernel's stores nor the neck pay for a
    layout change.  ``out``: optional contiguous [Nx, Ny, Nz, C(*T)] CUDA buffer to fill.
    ``channels_last=False`` runs the reference-layout kernel (contiguous [C, Nx, Ny, Nz])."""
    views = list(feats)
    for i, v in enumerate(views):
        _check_cuda(v, f'feats[{i}]')
    s = len(views)
    c, hf, wf = views[0].shape
    assert s == num_views * num_frames
    assert all(tuple(v.shape) == (c, hf, wf) for v in views)
    views = [v.contiguous() for v in views]
    table = (ctypes.c_void_p * s)(*[v.data_ptr() for v in views])
    dev = views[0].device
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
                          device=dev, dtype=torch.float32)
        capi.check(capi.lib().dfm_multiview_lift_views(
            ctypes.byref(desc), table,
            proj.ctypes.data_as(ctypes.c_void_p),
            img_w.ctypes.data_as(ctypes.c_void_p),
            ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(ys.data_ptr()),
            ctypes.c_void_p(zs.data_ptr()), _ptr(vol), _stream()),
            'dfm_multiview_lift_views')
        return vol
    shape_cl = (n_voxels[0], n_voxels[1], n_voxels[2], cout)
    if out is None:
        out = torch.empty(shape_cl, device=dev, dtype=torch.float32)
    assert tuple(out.shape) == shape_cl and out.is_contiguous() and out.is_cuda
    capi.check(capi.lib().dfm_multiview_lift_views_cl(
        ctypes.byref(desc), table,
        proj.ctypes.data_as(ctypes.c_void_p),
        img_w.ctypes.data_as(ctypes.c_void_p),
        ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(ys.data_ptr()),
        ctypes.c_void_p(zs.data_ptr()), _ptr(out), _stream()),
        'dfm_multiview_lift_views_cl')
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
        # batch_feats: [B, T*Nv, C, Hf, Wf], or per sample a list of T*Nv [C, Hf, Wf] views
        view0 = batch_feats[0][0]
        cout = view0.shape[0] * (num_frames if self.temporal_aggregate == 'concat' else 1)
        # one channels-last buffer for the batch; the reference-shaped view is returned
        buf = torch.empty((len(batch_feats), nvx[0], nvx[1], nvx[2], cout),
                          device=view0.device, dtype=torch.float32)
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


# ---------------------------------------------------------------------------------------------
# Per-view image-feature cache of the detectors
# ---------------------------------------------------------------------------------------------
_U64 = (1 << 64) - 1


def _view_fingerprints(batch):
    """[N, ...] contiguous fp32 CUDA views -> N hashable 128-bit fingerprints (one launch of
    ``dfm_view_fingerprint``, one device-to-host copy)."""
    n = batch.shape[0]
    out = torch.empty((n, 2), dtype=torch.int64, device=batch.device)
    capi.check(capi.lib().dfm_view_fingerprint(_ptr(batch), n, batch[0].numel(), _ptr(out),
                                               _stream()), 'dfm_view_fingerprint')
    return [(a & _U64, b & _U64) for a, b in out.cpu().tolist()]


def _views_equal(pairs):
    """[(a, b)] of equally shaped fp32 CUDA views -> [bool]: bitwise equality of each pair (one
    launch of ``dfm_views_equal``, one device-to-host copy)."""
    n = len(pairs)
    a = (ctypes.c_void_p * n)(*[x.data_ptr() for x, _ in pairs])
    b = (ctypes.c_void_p * n)(*[y.data_ptr() for _, y in pairs])
    mismatch = torch.empty(n, dtype=torch.int32, device=pairs[0][0].device)
    capi.check(capi.lib().dfm_views_equal(a, b, n, pairs[0][0].numel(), _ptr(mismatch),
                                          _stream()), 'dfm_views_equal')
    return [m == 0 for m in mismatch.cpu().tolist()]


def _as_batch(views):
    """Equally shaped contiguous views -> one [N, ...] tensor: a view of their storage when
    they lie back to back in it (a run of one ``img``), else a stacked copy."""
    v0 = views[0]
    step = v0.numel() * v0.element_size()
    if all(v.is_contiguous() and v.untyped_storage().data_ptr() == v0.untyped_storage().data_ptr()
           and v.data_ptr() == v0.data_ptr() + i * step for i, v in enumerate(views)):
        return torch.as_strided(v0, (len(views),) + tuple(v0.shape),
                                (v0.numel(),) + tuple(v0.stride()))
    return torch.stack(views)


class _ViewFeatureCache:
    """Image features of single input views, keyed by the view's exact content.

    An entry holds a copy of the view (callers may overwrite their input buffer), what the
    detector keeps of its features, and the state of the image modules it was computed under.
    The fingerprint only finds a candidate: a view is served from an entry only when it is
    bitwise equal to the entry's copy.  Least recently used entries go first; a hit refreshes
    its entry.  ``max_views`` counts entries."""

    def __init__(self, max_views):
        self.max_views = max_views
        self.entries = collections.OrderedDict()   # (shape, fingerprint) -> [view, feat, state]
        self.hits = self.misses = self.rejected = 0

    def clear(self):
        self.entries.clear()

    def stats(self):
        nbytes = sum(t.numel() * t.element_size() for e in self.entries.values() for t in e[:2])
        return dict(hits=self.hits, misses=self.misses, rejected=self.rejected,
                    views=len(self.entries), bytes=nbytes)

    def run(self, batch, compute, state, forced=()):
        """batch: [N, ...] contiguous views.  ``compute(views)`` returns, for a list of views,
        a list of ``(kept, extra)``: ``kept`` is stored, ``extra`` only handed back.  Views in
        ``forced`` are always computed (the caller needs their ``extra``).  Returns per view
        ``(kept, extra)``, ``extra`` None unless the view was computed in this call.  The
        missing views go to one ``compute`` call; a view equal to another view of the same call
        is computed once.  ``state(check)`` is the state of the modules that compute features
        (``check``: first empty the cache if a parameter upload is already due): entries
        recorded under another state are dropped, and new entries record the state after
        ``compute``."""
        views = list(batch)
        shape = tuple(batch.shape[1:])
        keys = [(shape,) + tuple(k) for k in _view_fingerprints(batch)]
        now = state(True)
        first = {}                    # key -> the view of this call that stands for it
        checks = []                   # (view index, the view it may equal, from the cache?)
        for i in sorted(range(len(views)), key=lambda i: i not in forced):
            k = keys[i]
            if k in first:
                checks.append((i, views[first[k]], False))
                continue
            first[k] = i
            e = self.entries.get(k)
            if e is not None and e[2] != now:
                del self.entries[k]
            elif e is not None and i not in forced:
                checks.append((i, e[0], True))
        equal = _views_equal([(views[i], other) for i, other, _ in checks]) if checks else []
        result = [None] * len(views)
        same_as = {}
        for (i, _, cached), ok in zip(checks, equal):
            if not ok:
                self.rejected += 1
            elif cached:
                self.entries.move_to_end(keys[i])
                result[i] = (self.entries[keys[i]][1], None)
            else:
                same_as[i] = first[keys[i]]
        todo = [i for i in range(len(views)) if result[i] is None and i not in same_as]
        if todo:
            for i, r in zip(todo, compute([views[i] for i in todo])):
                result[i] = r
            after = state(False)
            for i in todo:
                if first[keys[i]] == i:       # a colliding twin of this call is not kept
                    kept = result[i][0]
                    if kept.untyped_storage().nbytes() != kept.numel() * kept.element_size():
                        kept = kept.clone()   # a view into a batch would keep the whole batch
                    self.entries.pop(keys[i], None)
                    self.entries[keys[i]] = [views[i].clone(), kept, after]
            while len(self.entries) > self.max_views:
                self.entries.popitem(last=False)
        for i, j in same_as.items():
            result[i] = (result[j][0], None)
        self.hits += len(views) - len(todo)
        self.misses += len(todo)
        return result


# ---------------------------------------------------------------------------------------------
# Whole detectors: DfM (KITTI) and MultiViewDfM (Waymo), test path only
# ---------------------------------------------------------------------------------------------
def bbox3d2result(bboxes, scores, labels):
    """mmdet3d.core.bbox3d2result (core/bbox/transforms.py:53-76): results on the CPU."""
    return dict(boxes_3d=bboxes.to('cpu'), scores_3d=scores.cpu(), labels_3d=labels.cpu())


@DETECTORS.register_module()
class DfM(nn.Module):
    """The reference detector ``DfM`` (detectors/dfm.py:17-441) at test time, built from the
    shipped ``model`` dict (minus ``type``) with the local registries and the constructor's
    injections (:43-109).  The training-only entries (``lidar_model``, ``neck_2d``,
    ``bbox_head_2d``, ``depth_head_2d``, ``imitation_cfgs``) are accepted and not built;
    ``normalizer_clamp_value`` only reaches the LIGA head, as in the reference (:107-108)."""

    def __init__(self, backbone, neck, backbone_stereo, backbone_3d, bbox_head_3d, neck_2d=None,
                 neck_3d=None, feature_transformation=None, bbox_head_2d=None,
                 depth_head_2d=None, depth_head=None, lidar_model=None, depth_cfg=None,
                 voxel_cfg=None, normalizer_clamp_value=10, imitation_cfgs=None, train_cfg=None,
                 test_cfg=None, pretrained=None, init_cfg=None):
        super().__init__()
        from .registry import build_backbone, build_head, build_neck
        cp = copy.deepcopy
        self.backbone = build_backbone(cp(backbone))
        self.neck = build_neck(cp(neck))
        if backbone_stereo is not None:
            backbone_stereo = cp(backbone_stereo)
            if depth_cfg is not None:
                backbone_stereo.update(depth_cfg=depth_cfg)
            self.backbone_stereo = build_backbone(backbone_stereo)
        if backbone_3d is not None:
            self.backbone_3d = build_backbone(cp(backbone_3d))
        if neck_3d is not None:
            self.neck_3d = build_neck(cp(neck_3d))
        if feature_transformation is not None:
            feature_transformation = cp(feature_transformation)
            feature_transformation.update(cat_img_feature=self.neck.cat_img_feature,
                                          in_sem_channels=self.neck.sem_channels[-1])
            self.feature_transformation = build_neck(feature_transformation)
        if depth_head is not None:
            self.depth_head = build_head(cp(depth_head))
        self.imitation_cfgs = imitation_cfgs
        if depth_cfg is not None:
            self.downsampled_depth_offset = 0.5
            self.depth_downsample_factor = depth_cfg['downsample_factor']
            self.prepare_depth(depth_cfg)
            if feature_transformation is not None:
                self.feature_transformation.depth_cfg = depth_cfg
            if depth_head is not None:
                self.backbone_stereo.downsampled_depth = self.downsampled_depth
                self.depth_head.depth_samples = self.depth
                self.depth_head.downsample_factor = self.depth_downsample_factor
        if voxel_cfg is not None:
            self.prepare_coordinates_3d(voxel_cfg)
            if feature_transformation is not None:
                self.feature_transformation.coordinates_3d = self.coordinates_3d
        self.normalizer_clamp_value = normalizer_clamp_value
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        bbox_head_3d = cp(bbox_head_3d)
        bbox_head_3d.update(train_cfg=train_cfg, test_cfg=test_cfg)
        if bbox_head_3d['type'] == 'LIGAAnchor3DHead':
            bbox_head_3d.update(normalizer_clamp_value=normalizer_clamp_value)
        self.bbox_head_3d = build_head(bbox_head_3d)
        self._feature_cache = None

    # ---- per-view image-feature cache ----------------------------------------------------
    def set_feature_cache(self, max_views):
        """Reuse image features across ``simple_test`` calls, for video.  A view of ``img``
        whose content is bitwise equal to a view an earlier call computed (within the last
        ``max_views`` distinct views) takes that call's features instead of going through the
        image backbone and neck again; the results are bitwise those of a run without the
        cache.  DfM keeps the stereo feature's channels-last twin of each frame (current
        frames are always computed, previous frames are looked up); MultiViewDfM keeps FPN
        level 0 of every view of a multi-frame config (the single-frame camsync config never
        uses the cache).  ``0`` (the default) turns it off.  Every call empties the cache."""
        max_views = int(max_views)
        if max_views < 0:
            raise ValueError(f'max_views must be >= 0, got {max_views}')
        self._feature_cache = _ViewFeatureCache(max_views) if max_views else None

    def feature_cache_stats(self):
        """``dict(hits, misses, rejected, views, bytes)`` since ``set_feature_cache``: views
        served without computing / views computed / fingerprint matches that failed the
        bitwise check; entries held and their device bytes (view copies and features)."""
        c = self._feature_cache
        if c is None:
            return dict(hits=0, misses=0, rejected=0, views=0, bytes=0)
        return c.stats()

    def _feature_cache_state(self, device, check=True):
        """What cached features depend on besides the view: the image modules' parameter
        uploads and conv_impl, and the device.  With ``check``, an upload that is already due
        (``train()``, ``load_state_dict``, ``sync_params()``, a parameter written in place,
        replaced or moved) empties the cache at once."""
        mods = (self.backbone, self.neck)
        syncs = [getattr(m, '_sync', None) for m in mods]
        if check and any(sy is not None and sy.pending() for sy in syncs):
            self._feature_cache.clear()
        return (str(device),) + tuple((m.conv_impl, sy.generation if sy is not None else 0)
                                      for m, sy in zip(mods, syncs))

    def train(self, mode=True):
        if getattr(self, '_feature_cache', None) is not None:
            self._feature_cache.clear()
        return super().train(mode)

    @property
    def with_backbone_3d(self):
        return getattr(self, 'backbone_3d', None) is not None

    @property
    def with_neck_3d(self):
        return getattr(self, 'neck_3d', None) is not None

    @property
    def with_depth_head(self):
        return getattr(self, 'depth_head', None) is not None

    @property
    def with_depth_head_2d(self):
        return False   # the 2-D depth head is training-only and never built here

    def prepare_depth(self, depth_cfg):
        """dfm.py:152-168: the plane depths of the cost volume and the depth-bin centres."""
        assert depth_cfg['depth_min'] >= 0 and depth_cfg['depth_max'] > depth_cfg['depth_min']
        interval = (depth_cfg['depth_max'] - depth_cfg['depth_min']) / depth_cfg['num_bins']
        f = self.depth_downsample_factor
        self.downsampled_depth = torch.zeros(depth_cfg['num_bins'] // f, dtype=torch.float32)
        for i in range(depth_cfg['num_bins'] // f):
            self.downsampled_depth[i] = (i + self.downsampled_depth_offset) * f * interval + \
                depth_cfg['depth_min']
        self.depth = torch.zeros(depth_cfg['num_bins'], dtype=torch.float32)
        for i in range(depth_cfg['num_bins']):
            self.depth[i] = (i + 0.5) * interval + depth_cfg['depth_min']

    def prepare_coordinates_3d(self, voxel_cfg):
        """dfm.py:170-211 (sample_rate 1): the [Nz, Ny, Nx, 3] voxel-centre grid."""
        pcr, vs = voxel_cfg['point_cloud_range'], voxel_cfg['voxel_size']
        grid = (np.array(pcr[3:6], dtype=np.float32) - np.array(pcr[0:3], dtype=np.float32)) / \
            np.array(vs)
        nx, ny, nz = np.round(grid).astype(np.int64).tolist()
        zs = torch.linspace(pcr[2] + vs[2] / 2., pcr[5] - vs[2] / 2., nz, dtype=torch.float32)
        ys = torch.linspace(pcr[1] + vs[1] / 2., pcr[4] - vs[1] / 2., ny, dtype=torch.float32)
        xs = torch.linspace(pcr[0] + vs[0] / 2., pcr[3] - vs[0] / 2., nx, dtype=torch.float32)
        zs, ys, xs = torch.meshgrid(zs, ys, xs, indexing='ij')
        self.coordinates_3d = torch.stack([xs, ys, zs], dim=-1).float()

    def _check_test_input(self, img, img_metas, min_views):
        if self.training:
            raise RuntimeError(f'{type(self).__name__} runs the test path only: call .eval()')
        if img.dim() != 5 or img.shape[2] != 3 or img.shape[1] < min_views:
            raise ValueError(f'img must be [B, N >= {min_views}, 3, H, W], got '
                             f'{tuple(img.shape)}')
        if len(img_metas) != img.shape[0]:
            raise ValueError(f'{len(img_metas)} img_metas for a batch of {img.shape[0]}')
        _check_cuda(img, 'img')

    def extract_feat(self, img, img_metas):
        """dfm.py:264-298 for one sample (the stereo backbone takes B == 1).  The cur / prev
        pair goes through LIGAResNet in one call (eval BatchNorm: equal to two calls); the
        reference's device copy of ``cur2prevs`` stays a host tensor, which is what the stereo
        backbone reads, so no host synchronisation is added.  With the feature cache on, the
        previous frame's stereo feature may come from an earlier call."""
        pair = img[0, :2].contiguous()
        if self._feature_cache is None:
            feats = self.backbone(pair)
            cur_feats = [pair[0:1]] + [f[0:1] for f in feats]
            prev_feats = [pair[1:2]] + [f[1:2] for f in feats]
            cur_stereo_feat, cur_sem_feat = self.neck(cur_feats)
            prev_stereo_feat, _ = self.neck(prev_feats)      # prev semantic feature unused (:283)
        else:
            (cur_cl, cur_sem_feat), (prev_cl, _) = self._feature_cache.run(
                pair, self._stereo_twins, lambda check: self._feature_cache_state(img.device, check),
                forced=(0,))
        for meta in img_metas:
            c2p = meta['cur2prevs']
            if isinstance(c2p, torch.Tensor):   # e.g. metas already through extract_feat
                c2p = c2p.detach().cpu()
            meta['cur2prevs'] = torch.as_tensor(np.asarray(c2p, dtype=np.float64),
                                                dtype=img.dtype)
        if self._feature_cache is not None:
            costs, stereo_feats, mono_feats = self.backbone_stereo._forward_cl(
                cur_cl, prev_cl, img_metas)
        else:
            costs, stereo_feats, mono_feats = self.backbone_stereo(cur_stereo_feat,
                                                                   prev_stereo_feat, img_metas)
        return costs, stereo_feats, mono_feats, cur_sem_feat

    def _stereo_twins(self, views):
        """The feature function of DfM's cache: [3, H, W] views through LIGAResNet in one call
        and SPPUNetNeck one by one -> ``(stereo twin [H, W, 32], semantic feature)`` each."""
        x = _as_batch(views)
        feats = self.backbone(x)
        out = []
        for i in range(len(views)):
            stereo, sem = self.neck([x[i:i + 1]] + [f[i:i + 1] for f in feats])
            out.append((stereo._dfm_cl, sem))
        return out

    def _head_outputs(self, img, img_metas):
        """dfm.py:416-432 up to the head, sample by sample; DepthHead is fused into
        FrustumToVoxel (``CostLogits``), so no softmax volume is built."""
        outs = []
        for b in range(img.shape[0]):
            metas = img_metas[b:b + 1]
            costs, stereo_feats, _, cur_sem_feat = self.extract_feat(img[b:b + 1], metas)
            logits = CostLogits(costs, depth_samples=self.depth_head.depth_samples)
            volume_feat = self.feature_transformation(stereo_feats, logits, metas, cur_sem_feat)
            _, cv, nz, ny, nx = volume_feat.shape
            bev_feat = volume_feat.view(-1, cv * nz, ny, nx)          # height compression
            _, bev_feat = self.backbone_3d(bev_feat)
            outs.append(self.bbox_head_3d([bev_feat]))
        return tuple([torch.cat([o[k][0] for o in outs])] for k in range(3))

    def simple_test(self, img, img_metas):
        """dfm.py:416-441: ``[dict(boxes_3d, scores_3d, labels_3d, pseudo_lidar=True)]`` per
        sample.  ``img``: [B, N >= 2, 3, H, W] CUDA (current frame first)."""
        self._check_test_input(img, img_metas, 2)
        outs = self._head_outputs(img, img_metas)
        bbox_list = self.bbox_head_3d.get_bboxes(*outs, img_metas)
        results = [bbox3d2result(*r) for r in bbox_list]
        for r in results:
            r['pseudo_lidar'] = True
        return results

    def forward_test(self, img, img_metas, **kwargs):
        return self.simple_test(img, img_metas)


@DETECTORS.register_module()
class MultiViewDfM(MultiViewDfMFeatureTransformation, DfM):
    """The reference detector ``MultiViewDfM`` (detectors/multiview_dfm.py:12-341) at test time:
    ResNet + FPN over every view, the lifting of ``MultiViewDfMFeatureTransformation``, the
    3-D neck and ``Anchor3DHead``."""

    def __init__(self, backbone, neck, backbone_stereo, backbone_3d, neck_3d, bbox_head_3d,
                 voxel_size, anchor_generator, neck_2d=None, bbox_head_2d=None,
                 depth_head_2d=None, depth_head=None, train_cfg=None, test_cfg=None,
                 valid_sample=True, temporal_aggregate='mean', transform_depth=True,
                 pretrained=None, init_cfg=None):
        super().__init__(backbone=backbone, neck=neck, backbone_stereo=backbone_stereo,
                         backbone_3d=backbone_3d, neck_3d=neck_3d, bbox_head_3d=bbox_head_3d,
                         neck_2d=neck_2d, bbox_head_2d=bbox_head_2d,
                         depth_head_2d=depth_head_2d, depth_head=depth_head,
                         train_cfg=train_cfg, test_cfg=test_cfg, pretrained=pretrained,
                         init_cfg=init_cfg)
        self.voxel_size = voxel_size
        self.voxel_range = anchor_generator['ranges'][0]
        self.n_voxels = [round((self.voxel_range[3 + a] - self.voxel_range[a]) / voxel_size[a])
                         for a in range(3)]
        self.anchor_generator_cfg = anchor_generator
        self.valid_sample = valid_sample
        self.temporal_aggregate = temporal_aggregate
        self.transform_depth = transform_depth

    def extract_feat(self, img, img_metas):
        """multiview_dfm.py:67-117.  Every view of every sample, current and previous, goes
        through ResNet and FPN in one call; per sample the views stay in the reference's
        current-then-previous order."""
        batch_size, _, c_in, h, w = img.shape
        num_views = img_metas[0]['num_views']
        num_ref_frames = img_metas[0]['num_ref_frames']
        num_frames = num_ref_frames + 1 if num_ref_frames > 0 else 1
        if img.shape[1] != num_views * num_frames:
            raise ValueError(f'img has {img.shape[1]} views, the metas say {num_views} x '
                             f'{num_frames}')
        input_shape = img.shape[-2:]
        for img_meta in img_metas:
            img_meta.update(input_shape=input_shape)
        if self._feature_cache is not None and num_frames > 1:
            got = self._feature_cache.run(
                img.reshape(-1, c_in, h, w).contiguous(), self._fpn_level0,
                lambda check: self._feature_cache_state(img.device, check))
            s = img.shape[1]
            batch_feats = [[got[b * s + j][0] for j in range(s)] for b in range(batch_size)]
            return self.feature_transformation(batch_feats, img_metas, num_views, num_frames)
        feats = self.neck(self.backbone(img.reshape(-1, c_in, h, w)))[0]
        _, c_feat, h_feat, w_feat = feats.shape
        batch_feats = feats.view(batch_size, -1, c_feat, h_feat, w_feat)
        return self.feature_transformation(batch_feats, img_metas, num_views, num_frames)

    def _fpn_level0(self, views):
        """The feature function of MultiViewDfM's cache: views through ResNet and FPN in one
        call -> FPN level 0 ``[64, H/4, W/4]`` of each."""
        f0 = self.neck(self.backbone(_as_batch(views)))[0]
        return [(f0[i], None) for i in range(len(views))]

    def simple_test(self, img, img_metas):
        """multiview_dfm.py:321-341: ``[dict(boxes_3d, scores_3d, labels_3d)]`` per sample.
        ``img``: [B, Nv * T, 3, H, W] CUDA, current views first."""
        self._check_test_input(img, img_metas, 1)
        bev_feat = self.extract_feat(img, img_metas)[0]
        outs = self.bbox_head_3d([bev_feat])
        bbox_list = self.bbox_head_3d.get_bboxes(*outs, img_metas)
        return [bbox3d2result(*r) for r in bbox_list]
