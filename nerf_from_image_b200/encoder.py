"""Regression heads of the bootstrap encoder on sm_90a (``include/nfi_encoder.h``).

Encoder training (the reference's ``train_coord_regressor``, run.py:1521-1706) runs
``BootstrapEncoder`` (models/encoder.py) forward and backward in eager fp32 every iteration.  Almost
all of its arithmetic is in the heads behind the SegFormer backbone: ``post`` (two 512-channel 3x3
convs and a 512 -> 4 one on the x4-upsampled features) and ``w_regressor_pre`` (a 512-channel 3x3
conv at the backbone's resolution).  ``enable_fused_encoder`` switches a reference
``BootstrapEncoder`` instance to a forward with the same contract, ``(coords, segmentation, w)``:

- the backbone(s) run as they are, eagerly;
- from their output(s) to ``maps`` (``post``'s output) and ``pooled`` (the spatial mean of
  ``relu(w_regressor_pre(relu(features_latent)))``) one autograd function runs
  ``nfi_encoder_forward`` and, in its backward, ``nfi_encoder_backward``: gradients to the
  features and to the eight weights and biases of ``post[0]``, ``post[2]``, ``post[4]`` and
  ``w_regressor_pre[0]``;
- the sigmoid of the mask channel and ``w_regressor_post`` (two Linear layers on [B,512]) run in
  torch.

The binding is one line after the module is built, before ``nn.DataParallel``::

    enable_fused_encoder(coord_regressor)

The instance's class is swapped for a subclass that overrides ``forward``, so ``nn.DataParallel``'s
replicas run the fused forward too, and the parameters, their names and ``state_dict()`` are the
module's own: checkpoints interchange with unfused runs, and the parameters are read on every call,
so optimiser updates take effect.  Under ``torch.no_grad()`` nothing is kept for a backward.  Refused
with ``NfiError``, with no fallback: CPU or non-fp32 tensors, heads not laid out as
encoder.py:50-68, sizes outside the kernels' envelope, a gradient through an eval-mode call, a
double backward (``create_graph``) and a second backward of one forward.
"""
import ctypes

import torch
from torch import nn

from . import _lib

CHANNELS = 512
MAPS = _lib.ENCODER_MAPS
SCALE = 4   # SegFormer's output is 1/4 of the image (encoder.py:75-80)


def _conv_ok(m, cin, cout):
    return (isinstance(m, nn.Conv2d) and type(m).forward is nn.Conv2d.forward
            and m.in_channels == cin and m.out_channels == cout
            and m.kernel_size == (3, 3) and m.stride == (1, 1) and m.padding == (1, 1)
            and m.dilation == (1, 1) and m.groups == 1 and m.bias is not None
            and m.padding_mode == 'zeros')


def _relu_ok(m):
    return type(m) is nn.ReLU


def head_convs(enc):
    """(post[0], post[2], post[4], w_regressor_pre[0]) of a module laid out as the reference's
    ``BootstrapEncoder`` (encoder.py:50-68), None for a head it does not have; raises NfiError
    otherwise."""
    pose, latent = bool(getattr(enc, 'pose_regressor', False)), bool(getattr(enc, 'latent_regressor', False))
    convs = [None] * 4
    if pose:
        post = getattr(enc, 'post', None)
        if not (isinstance(post, nn.Sequential) and len(post) == 5 and _conv_ok(post[0], CHANNELS, CHANNELS)
                and _relu_ok(post[1]) and _conv_ok(post[2], CHANNELS, CHANNELS) and _relu_ok(post[3])
                and _conv_ok(post[4], CHANNELS, MAPS)):
            raise _lib.NfiError('fused encoder: post must be Conv2d(512, 512, 3, padding=1), ReLU, '
                                'Conv2d(512, 512, 3, padding=1), ReLU, Conv2d(512, 4, 3, padding=1) '
                                '(encoder.py:50-56)')
        convs[0:3] = post[0], post[2], post[4]
    if latent:
        pre = getattr(enc, 'w_regressor_pre', None)
        if not (isinstance(pre, nn.Sequential) and len(pre) == 2 and _conv_ok(pre[0], CHANNELS, CHANNELS)
                and _relu_ok(pre[1])):
            raise _lib.NfiError('fused encoder: w_regressor_pre must be Conv2d(512, 512, 3, padding=1), '
                                'ReLU (encoder.py:58-61)')
        convs[3] = pre[0]
    if not (pose or latent):
        raise _lib.NfiError('fused encoder: the module has neither head')
    if getattr(enc, 'separate_backbones', False) and not hasattr(enc, 'backbone_latent'):
        raise _lib.NfiError('fused encoder: separate_backbones without backbone_latent')
    return convs


def heads(enc, features, features_latent):
    """(maps [B,4h,4w,4] channel-last, pooled [B,512]) of the heads of ``enc`` from the backbone
    output(s) [B,512,h,w]; ``features_latent`` may be ``features`` (one backbone), and either is
    None without its head (its output is then an empty tensor)."""
    convs = head_convs(enc)
    pose, latent = convs[0] is not None, convs[3] is not None
    if (features is None) == pose or (features_latent is None) == latent:
        raise _lib.NfiError('fused encoder: features for exactly the heads the module has')
    shared = pose and latent and features_latent is features
    ws = []
    for c in convs:
        ws += [c.weight, c.bias] if c is not None else [None, None]
    tensors = [t for t in [features, features_latent] + ws if t is not None]
    needs = torch.is_grad_enabled() and any(t.requires_grad for t in tensors)
    if needs and not enc.training:
        raise _lib.NfiError('fused encoder: no backward through an eval-mode call (run it under '
                            'torch.no_grad(), or in train mode)')
    return _HeadsFunction.apply(features, None if shared else features_latent, shared, int(needs), *ws)


class _HeadsFunction(torch.autograd.Function):
    """(features, features_latent or None, shared, save, 8 weights / biases) -> (maps, pooled)."""

    @staticmethod
    def forward(ctx, feat, feat_l, shared, save, *ws):
        pose, latent = feat is not None, (feat_l is not None or shared)
        src = feat if feat is not None else feat_l
        tensors = [t for t in (feat, feat_l) + ws if t is not None]
        if not all(t.is_cuda for t in tensors):
            raise _lib.NfiError('fused encoder: only runs on CUDA tensors (there is no CPU path)')
        if not all(t.dtype == torch.float32 for t in tensors):
            raise _lib.NfiError('fused encoder: fp32 features and parameters only, got %s'
                                % sorted({str(t.dtype) for t in tensors}))
        dev = src.device
        if any(t.device != dev for t in tensors):
            raise _lib.NfiError('fused encoder: features and parameters on different devices')
        if src.dim() != 4 or src.shape[1] != CHANNELS or any(
                t is not None and t.shape != src.shape for t in (feat, feat_l)):
            raise _lib.NfiError('fused encoder: features must be [B,512,h,w] (both backbones alike), '
                                'got %s' % [tuple(t.shape) for t in (feat, feat_l) if t is not None])
        B, C, h, w = src.shape
        lib = _lib.load()
        with torch.cuda.device(dev):
            fc = feat.detach().contiguous() if pose else None
            flc = (fc if shared else feat_l.detach().contiguous()) if latent else None
            wc = [t.detach().contiguous() if t is not None else None for t in ws]
            maps = torch.empty(B, SCALE * h, SCALE * w, MAPS, device=dev) if pose else torch.empty(0, device=dev)
            pooled = torch.empty(B, C, device=dev) if latent else torch.empty(0, device=dev)
            p = _lib.EncoderParams()
            p.batch, p.height, p.width, p.channels = B, h, w, C
            p.pose_regressor, p.latent_regressor, p.save = int(pose), int(latent), save
            p.features, p.features_latent = _lib.ptr(fc), _lib.ptr(flc)
            (p.post0_w, p.post0_b, p.post2_w, p.post2_b, p.post4_w, p.post4_b, p.wpre_w,
             p.wpre_b) = [_lib.ptr(t) for t in wc]
            p.maps, p.pooled = (_lib.ptr(maps) if pose else None), (_lib.ptr(pooled) if latent else None)
            nbytes = lib.nfi_encoder_workspace_bytes(ctypes.byref(p))
            if nbytes == 0:
                raise _lib.NfiError('fused encoder: sizes outside the kernels\' envelope (B %d, features '
                                    '%d x %d, %d channels)' % (B, h, w, C))
            work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            p.workspace, p.workspace_bytes = work.data_ptr(), nbytes
            stream = _lib.stream(dev)
            _lib.check(lib.nfi_encoder_forward(ctypes.byref(p), stream))
        # the backward reads the workspace and the tensors behind p's pointers
        ctx.state = (p, work, fc, flc, wc) if save else None
        ctx.shared = shared
        return maps, pooled

    @staticmethod
    def backward(ctx, g_maps, g_pooled):
        p, work, fc, flc, wc = _lib.take_saved(ctx, 'encoder')
        needs = ctx.needs_input_grad
        dev = work.device
        with torch.cuda.device(dev):
            gf = torch.zeros_like(fc) if (fc is not None and needs[0]) else None
            gfl = torch.zeros_like(flc) if (needs[1] and not ctx.shared) else None
            gw = [torch.zeros_like(t) if (t is not None and needs[4 + i]) else None for i, t in enumerate(wc)]
            g = _lib.EncoderGrads()
            g.g_features = _lib.ptr(gf)
            g.g_features_latent = _lib.ptr(gf) if ctx.shared else _lib.ptr(gfl)
            (g.g_post0_w, g.g_post0_b, g.g_post2_w, g.g_post2_b, g.g_post4_w, g.g_post4_b, g.g_wpre_w,
             g.g_wpre_b) = [_lib.ptr(t) for t in gw]
            gm = g_maps.to(torch.float32).contiguous() if p.pose_regressor else None
            gp = g_pooled.to(torch.float32).contiguous() if p.latent_regressor else None
            _lib.check(_lib.load().nfi_encoder_backward(ctypes.byref(p), _lib.ptr(gm), _lib.ptr(gp),
                                                        ctypes.byref(g), _lib.stream(dev)))
        del p, work
        return (gf, gfl, None, None, *gw)


def saved_activations(out):
    """The post-ReLU activations kept by the saved forward behind ``out`` (``maps`` or ``pooled`` of
    a call that requires grad, before its backward has run), fp32 channel-last: a dict of
    'x0', 'a1', 'a2' [B,4h,4w,512] (pose head) and 'xl', 'al' [B,h,w,512] (latent head).  Where a
    value is positive the backward takes the ReLU's pass branch; tests read the branches from them."""
    p, work = _lib.find_saved(out, 'encoder')[:2]
    dev = work.device
    lib = _lib.load()
    B, h, w, C = p.batch, p.height, p.width, p.channels
    names = []
    if p.pose_regressor:
        names += [(0, 'x0', SCALE), (1, 'a1', SCALE), (2, 'a2', SCALE)]
    if p.latent_regressor:
        names += [(3, 'xl', 1), (4, 'al', 1)]
    res = {}
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)
        for layer, name, s in names:
            t = torch.empty(B, s * h, s * w, C, device=dev)
            _lib.check(lib.nfi_encoder_saved_activation(ctypes.byref(p), layer, _lib.ptr(t), stream))
            res[name] = t
    return res


def _fused_forward(self, x):
    """BootstrapEncoder.forward (encoder.py:70-103) with the heads on nfi_encoder_forward."""
    features = self.backbone(x)
    features_latent = None
    if self.latent_regressor:
        features_latent = self.backbone_latent(x) if self.separate_backbones else features
    maps, pooled = heads(self, features if self.pose_regressor else None, features_latent)
    coords = segmentation = w = None
    if self.pose_regressor:
        coords = maps[..., :3]
        segmentation = torch.sigmoid(maps[..., 3])
    if self.latent_regressor:
        w = self.w_regressor_post(pooled).unsqueeze(1)
    return coords, segmentation, w


def enable_fused_encoder(bootstrap_encoder, enabled=True):
    """Switches a reference ``BootstrapEncoder`` instance to the fused heads (``enabled=False``
    switches it back).  Checks the heads' layout now; returns the instance."""
    if enabled:
        head_convs(bootstrap_encoder)
    return _lib.switch_class(bootstrap_encoder, _fused_forward, enabled)
