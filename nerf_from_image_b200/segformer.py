"""The bootstrap encoder's SegFormer-B5 backbone on sm_90a (``include/nfi_segformer.h``).

Encoder training (the reference's ``train_coord_regressor``, run.py:1521-1706) runs the SegFormer
backbone (models/segformer.py:175-275) forward and backward in eager fp32 every iteration.
``enable_fused_segformer`` switches a reference ``Segformer`` instance to a forward with the same
contract, image [B,3,H,H] -> features [B,out_features,H/4,H/4], on ``nfi_segformer_forward``, and
its backward (to every parameter; there is no image gradient) on ``nfi_segformer_backward``::

    enable_fused_segformer(coord_regressor.backbone)
    enable_fused_segformer(coord_regressor.backbone_latent)   # with separate_backbones

The instance's class is swapped for a subclass that overrides ``forward``, so ``nn.DataParallel``'s
replicas run the fused forward too, and the parameters, their names and ``state_dict()`` are the
module's own.  In train mode the drop-path masks are drawn by the module's own ``SegDropPath``
modules, in block order, attention branch before MLP branch, exactly as its forward draws them, so
the masks and the generator's state match an eager forward from the same seed.  Under
``torch.no_grad()`` nothing is kept for a backward.  Refused with ``NfiError``, with no fallback:
CPU or non-fp32 tensors, a module not laid out as the reference's B5 (any depths, out_features a
multiple of 64), images that are not square, not a multiple of 32 or larger than 256, an image that
requires grad, a double backward (``create_graph``) and a second backward of one forward.
"""
import ctypes

import torch
from torch import nn

from . import _lib

DIMS = (64, 128, 320, 512)
HEADS = (1, 2, 5, 8)
SR = (8, 4, 2, 1)
DECODER = _lib.SEGFORMER_DECODER
MAX_DEPTH = _lib.SEGFORMER_MAX_DEPTH


def _is(m, cls):
    return type(m) is cls


def _linear_ok(m, cin, cout):
    return _is(m, nn.Linear) and m.in_features == cin and m.out_features == cout and m.bias is not None


def _ln_ok(m, c, eps):
    return (_is(m, nn.LayerNorm) and tuple(m.normalized_shape) == (c,) and m.eps == eps
            and m.weight is not None and m.bias is not None)


def _conv_ok(m, cin, cout, k, stride, pad, groups=1):
    return (_is(m, nn.Conv2d) and m.in_channels == cin and m.out_channels == cout
            and m.kernel_size == (k, k) and m.stride == (stride, stride) and m.padding == (pad, pad)
            and m.dilation == (1, 1) and m.groups == groups and m.bias is not None
            and m.padding_mode == 'zeros')


def _block_ok(blk, C, heads, sr):
    a, mlp = getattr(blk, 'attn', None), getattr(blk, 'mlp', None)
    if a is None or mlp is None or not hasattr(blk, 'drop_path'):
        return False
    if not (_ln_ok(getattr(blk, 'norm1', None), C, 1e-6) and _ln_ok(getattr(blk, 'norm2', None), C, 1e-6)):
        return False
    if not (getattr(a, 'num_heads', None) == heads and getattr(a, 'sr_ratio', None) == sr
            and abs(getattr(a, 'scale', 0) - 0.125) < 1e-12 and _linear_ok(a.q, C, C)
            and _linear_ok(a.kv, C, 2 * C) and _linear_ok(a.proj, C, C)):
        return False
    if sr > 1 and not (_conv_ok(getattr(a, 'sr', None), C, C, sr, sr, 0)
                       and _ln_ok(getattr(a, 'norm', None), C, 1e-5)):
        return False
    if sr == 1 and (hasattr(a, 'sr') or hasattr(a, 'norm')):
        return False
    dw = getattr(getattr(mlp, 'dwconv', None), 'dwconv', None)
    return (_linear_ok(mlp.fc1, C, 4 * C) and _linear_ok(mlp.fc2, 4 * C, C)
            and _conv_ok(dw, 4 * C, 4 * C, 3, 1, 1, groups=4 * C)
            and type(mlp.gelu) is nn.GELU and mlp.gelu.approximate == 'none')


def layout(m):
    """(depths, out_features) of a module laid out as the reference's B5 ``Segformer``
    (segformer.py:175-275); raises NfiError otherwise."""
    depths = []
    for i in range(4):
        C, Cp = DIMS[i], (3 if i == 0 else DIMS[i - 1])
        pe = getattr(m, 'patch_embed%d' % (i + 1), None)
        k, st, pad = (7, 4, 3) if i == 0 else (3, 2, 1)
        if pe is None or not (_conv_ok(getattr(pe, 'proj', None), Cp, C, k, st, pad)
                              and _ln_ok(getattr(pe, 'norm', None), C, 1e-5)):
            raise _lib.NfiError('fused segformer: patch_embed%d must be Conv2d(%d, %d, %d, stride %d, padding '
                                '%d), LayerNorm(%d) (segformer.py:131-161)' % (i + 1, Cp, C, k, st, pad, C))
        blocks = getattr(m, 'block%d' % (i + 1), None)
        if not isinstance(blocks, nn.ModuleList) or not 1 <= len(blocks) <= MAX_DEPTH:
            raise _lib.NfiError('fused segformer: block%d must be a ModuleList of 1..%d blocks'
                                % (i + 1, MAX_DEPTH))
        for j, blk in enumerate(blocks):
            if not _block_ok(blk, C, HEADS[i], SR[i]):
                raise _lib.NfiError('fused segformer: block%d.%d is not a SegBlock(%d, heads %d, mlp ratio 4, '
                                    'sr %d) (segformer.py:114-128)' % (i + 1, j, C, HEADS[i], SR[i]))
        if not _ln_ok(getattr(m, 'norm%d' % (i + 1), None), C, 1e-6):
            raise _lib.NfiError('fused segformer: norm%d must be LayerNorm(%d, eps=1e-6)' % (i + 1, C))
        lc = getattr(getattr(m, 'linear_c%d' % (i + 1), None), 'proj', None)
        if not _linear_ok(lc, C, DECODER):
            raise _lib.NfiError('fused segformer: linear_c%d must project %d -> %d' % (i + 1, C, DECODER))
        depths.append(len(blocks))
    fuse, pred = getattr(m, 'linear_fuse', None), getattr(m, 'linear_pred', None)
    if not _conv_ok(fuse, 4 * DECODER, DECODER, 1, 1, 0):
        raise _lib.NfiError('fused segformer: linear_fuse must be Conv2d(3072, 768, 1)')
    if pred is None or not (_conv_ok(pred, DECODER, pred.out_channels, 1, 1, 0) and pred.out_channels % 64 == 0
                            and 64 <= pred.out_channels <= 4096):
        raise _lib.NfiError('fused segformer: linear_pred must be Conv2d(768, out, 1) with out a multiple of 64 '
                            'in 64..4096')
    return tuple(depths), pred.out_channels


def param_names(depths):
    """The names of the module's parameters in ``named_parameters()`` order (nfi_segformer.h)."""
    names = []
    for i in range(4):
        names += ['patch_embed%d.%s' % (i + 1, n) for n in ('proj.weight', 'proj.bias', 'norm.weight', 'norm.bias')]
    for i in range(4):
        layers = (['norm1', 'attn.q', 'attn.kv', 'attn.proj'] + (['attn.sr', 'attn.norm'] if SR[i] > 1 else [])
                  + ['norm2', 'mlp.fc1', 'mlp.dwconv.dwconv', 'mlp.fc2'])
        for j in range(depths[i]):
            names += ['block%d.%d.%s.%s' % (i + 1, j, n, t) for n in layers for t in ('weight', 'bias')]
        names += ['norm%d.weight' % (i + 1), 'norm%d.bias' % (i + 1)]
    for i in reversed(range(4)):
        names += ['linear_c%d.proj.weight' % (i + 1), 'linear_c%d.proj.bias' % (i + 1)]
    return names + ['linear_fuse.weight', 'linear_fuse.bias', 'linear_pred.weight', 'linear_pred.bias']


def parameters_of(m, depths):
    """The parameter tensors in that order, read by attribute (an ``nn.DataParallel`` replica
    registers none)."""
    out = []
    for n in param_names(depths):
        t = m
        for part in n.split('.'):
            t = getattr(t, part)
        out.append(t)
    return out


def drop_scales(m, B, device, dtype=torch.float32):
    """The drop-path scales of one forward, [2 * blocks, B] (row 2k block k's attention branch, row
    2k + 1 its MLP branch), drawn by the module's own ``drop_path`` in its forward's order; None in
    eval mode (every scale 1, and the module draws nothing).  ``dtype`` is the forward's: the draws
    depend on it."""
    if not m.training:
        return None
    rows = []
    for i in range(4):
        for blk in getattr(m, 'block%d' % (i + 1)):
            for _ in range(2):
                rows.append(blk.drop_path(torch.ones(B, 1, 1, device=device, dtype=dtype)).reshape(B))
    return torch.stack(rows).contiguous()


def _check_tensors(img, params):
    tensors = [img] + list(params)
    if not all(t.is_cuda for t in tensors):
        raise _lib.NfiError('fused segformer: only runs on CUDA tensors (there is no CPU path)')
    if not all(t.dtype == torch.float32 for t in tensors):
        raise _lib.NfiError('fused segformer: fp32 image and parameters only, got %s'
                            % sorted({str(t.dtype) for t in tensors}))
    if any(t.device != img.device for t in tensors):
        raise _lib.NfiError('fused segformer: image and parameters on different devices')


class _SegformerFunction(torch.autograd.Function):
    """(image, drop-path scales or None, depths, save, *parameters) -> features."""

    @staticmethod
    def forward(ctx, img, scales, depths, save, *params):
        _check_tensors(img, params)
        dev = img.device
        B, _, H, W = img.shape
        out = params[-2].shape[0]
        lib = _lib.load()
        with torch.cuda.device(dev):
            ic = img.detach().contiguous()
            pc = [t.detach().contiguous() for t in params]
            feats = torch.empty(B, out, H // 4, W // 4, device=dev)
            p = _lib.SegformerParams()
            p.batch, p.height, p.width = B, H, W
            p.depths[:] = list(depths)
            p.out_features, p.save = out, save
            p.image = ic.data_ptr()
            arr = (ctypes.c_void_p * len(pc))(*[t.data_ptr() for t in pc])
            p.params = ctypes.cast(arr, ctypes.c_void_p)
            p.drop_scales = scales.data_ptr() if scales is not None else None
            p.features = feats.data_ptr()
            nbytes = lib.nfi_segformer_workspace_bytes(ctypes.byref(p))
            if nbytes == 0:
                raise _lib.NfiError('fused segformer: sizes outside the kernels\' envelope (B %d, %d x %d, '
                                    'depths %s, out %d)' % (B, H, W, tuple(depths), out))
            work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            p.workspace, p.workspace_bytes = work.data_ptr(), nbytes
            _lib.check(lib.nfi_segformer_forward(ctypes.byref(p), _lib.stream(dev)))
        # the backward reads the workspace and the tensors behind p's pointers
        ctx.state = (p, arr, work, ic, pc, scales) if save else None
        return feats

    @staticmethod
    def backward(ctx, g):
        p, arr, work, ic, pc, scales = _lib.take_saved(ctx, 'segformer')
        needs = ctx.needs_input_grad[4:]
        dev = work.device
        with torch.cuda.device(dev):
            # one zeroed buffer for every requested gradient (one memset, not one per tensor)
            sizes = [t.numel() if n else 0 for t, n in zip(pc, needs)]
            flat = torch.zeros(sum(sizes), device=dev)
            grads, off = [], 0
            for t, n, k in zip(pc, needs, sizes):
                grads.append(flat[off:off + k].view_as(t) if n else None)
                off += k
            garr = (ctypes.c_void_p * len(pc))(*[t.data_ptr() if t is not None else None for t in grads])
            gc = g.to(torch.float32).contiguous()
            _lib.check(_lib.load().nfi_segformer_backward(ctypes.byref(p), gc.data_ptr(), garr,
                                                          _lib.stream(dev)))
        del p, arr, work
        return (None, None, None, None, *grads)


def segformer(m, x):
    """``Segformer.forward`` (segformer.py:245-275) of ``m`` on ``x`` on the kernels."""
    depths, _ = layout(m)
    if not (torch.is_tensor(x) and x.dim() == 4 and x.shape[1] == 3 and x.shape[2] == x.shape[3]
            and x.shape[2] % 32 == 0 and 32 <= x.shape[2] <= 256):
        raise _lib.NfiError('fused segformer: images must be [B,3,H,H] with H a multiple of 32 in 32..256, '
                            'got %s' % (str(tuple(x.shape)) if torch.is_tensor(x) else type(x),))
    if x.requires_grad:
        raise _lib.NfiError('fused segformer: no gradient to the image (it must not require grad)')
    params = parameters_of(m, depths)
    _check_tensors(x, params)   # before the draw: a refused call leaves the generator as it was
    scales = drop_scales(m, x.shape[0], x.device)
    needs = torch.is_grad_enabled() and any(t.requires_grad for t in params)
    return _SegformerFunction.apply(x, scales, depths, int(needs), *params)


def _fused_forward(self, x):
    return segformer(self, x)


def enable_fused_segformer(module, enabled=True):
    """Switches a reference ``Segformer`` instance to the fused forward (``enabled=False`` switches it
    back).  Checks the layout now; returns the instance."""
    if enabled:
        layout(module)
    return _lib.switch_class(module, _fused_forward, enabled)
