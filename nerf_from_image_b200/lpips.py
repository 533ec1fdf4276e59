"""LPIPS-VGG distance of the inversion loss on sm_90a (``include/nfi_lpips.h``).

The reference's ``lib/metrics.py:97-137`` (``LPIPSLoss`` over ``lpips.LPIPS(net='vgg')``) runs the
VGG16 feature stack in eager fp32 on the image and on the target, 16 copies of each per inversion
image (``run.py:2202-2254``), then backpropagates into the image.  ``FusedLPIPS`` takes such a
module's weights and computes the same distance with ``nfi_lpips_forward`` (conv1_2 .. conv5_3 on
the synthesis network's wgmma kernel, conv1_1, pools and the head on small kernels of their own),
and its gradients to ``in0`` and, where it requires grad, ``in1`` with ``nfi_lpips_backward``.
The binding is one line in ``run.py``::

    loss_fn_lpips = FusedLPIPS(metrics.LPIPSLoss().to(device))

Only the two-tensor form every ``run.py`` call site uses is served.  ``in1`` may require grad: the
inversion step's augmented targets do (``optimize_iter`` grid-samples the prediction and the target
as one tensor, run.py:2217-2230), and their gradient is computed like ``in0``'s, by one backward
over both halves.  Everything else raises ``NfiError``: ``in1=None`` or cached-feature tuples, a
weight that requires grad, a second or double backward, CPU tensors, and sizes that are not
multiples of 16.  There is no CPU path and no fallback.
"""
import ctypes

import torch
from torch import nn

from . import _lib

# conv layers of lpips.pretrained_networks.vgg16: features [0:4], [4:9], [9:16], [16:23], [23:30]
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256),
                 (256, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
TAP_CHANNELS = (64, 128, 256, 512, 512)


def extract_weights(lpips_loss):
    """(shift [3], scale [3], [13 conv weights], [13 conv biases], [5 lin weights [C]]) of a module
    laid out as the reference's ``LPIPSLoss``: ``.lpips.scaling_layer.shift / .scale``, the Conv2d
    modules of ``.lpips.net.slice1 .. slice5`` in order, ``.lpips.lins[l].model[-1].weight``."""
    net = lpips_loss.lpips
    convs = [m for k in range(1, 6) for m in getattr(net.net, 'slice%d' % k).modules()
             if isinstance(m, nn.Conv2d)]
    got = tuple((c.in_channels, c.out_channels) for c in convs)
    if got != CONV_CHANNELS or any(c.kernel_size != (3, 3) or c.stride != (1, 1) or c.padding != (1, 1)
                                   or c.bias is None for c in convs):
        raise _lib.NfiError('FusedLPIPS serves the VGG16 network of lpips.LPIPS(net=\'vgg\') only; '
                            'got convs %s' % (got,))
    lins = [net.lins[k].model[-1].weight for k in range(5)]
    if tuple(w.numel() for w in lins) != TAP_CHANNELS:
        raise _lib.NfiError('FusedLPIPS: lin layers of %s channels' % ([w.numel() for w in lins],))
    return (net.scaling_layer.shift.reshape(3), net.scaling_layer.scale.reshape(3),
            [c.weight for c in convs], [c.bias for c in convs], [w.reshape(-1) for w in lins])


class FusedLPIPS(nn.Module):
    """Drop-in for the reference's ``LPIPSLoss`` in ``forward(in0, in1, normalize, reduction)``.

    The weights are copied into buffers, so ``.to()`` and ``nn.DataParallel`` replication carry
    them.  The distance is differentiable in ``in0`` and ``in1``, not in the weights."""

    def __init__(self, lpips_loss):
        super().__init__()
        shift, scale, cw, cb, lw = extract_weights(lpips_loss)
        f32 = lambda t: t.detach().to(torch.float32).contiguous().clone()
        self.register_buffer('shift', f32(shift))
        self.register_buffer('scale', f32(scale))
        for i in range(len(cw)):
            self.register_buffer('conv%d_weight' % i, f32(cw[i]))
            self.register_buffer('conv%d_bias' % i, f32(cb[i]))
        for i in range(len(lw)):
            self.register_buffer('lin%d_weight' % i, f32(lw[i]))

    def weights(self):
        return ([self.shift, self.scale]
                + [getattr(self, 'conv%d_weight' % i) for i in range(len(CONV_CHANNELS))]
                + [getattr(self, 'conv%d_bias' % i) for i in range(len(CONV_CHANNELS))]
                + [getattr(self, 'lin%d_weight' % i) for i in range(len(TAP_CHANNELS))])

    def forward(self, in0, in1=None, normalize=False, reduction='none'):
        if in1 is None or isinstance(in1, tuple):
            raise _lib.NfiError('FusedLPIPS serves the two-image form only (no feature output, no '
                                'cached features)')
        if normalize:
            _range_check(in0)
            _range_check(in1)
            in0 = 2 * in0 - 1
            in1 = 2 * in1 - 1
        # 0: distance only; 1: keep what the backward to in0 reads; 2: room for in1's gradient too
        save = 0
        if torch.is_grad_enabled() and (in0.requires_grad or in1.requires_grad):
            save = 2 if in1.requires_grad else 1
        out = _LpipsFunction.apply(in0, in1, self, save)[:, None]   # [N, 1]: lin(.).mean([2, 3]) summed
        if reduction == 'mean':
            return out.mean()
        return out


def _range_check(im):  # lib/metrics.py:22-27
    with torch.no_grad():
        eps = 1e-1
        assert im.max() < 1 + eps, 'Range check failed'
        assert im.min() > -eps, 'Range check failed'


def _params(m, in0, in1, out, save):
    ws = m.weights()
    p = _lib.LpipsParams()
    p.n, p.height, p.width, p.save = in0.shape[0], in0.shape[2], in0.shape[3], save
    p.in0, p.in1, p.out = _lib.ptr(in0), _lib.ptr(in1), _lib.ptr(out)
    p.shift, p.scale = _lib.ptr(ws[0]), _lib.ptr(ws[1])
    n = len(CONV_CHANNELS)
    for i in range(n):
        p.conv_w[i] = ws[2 + i].data_ptr()
        p.conv_b[i] = ws[2 + n + i].data_ptr()
    for i in range(len(TAP_CHANNELS)):
        p.lin_w[i] = ws[2 + 2 * n + i].data_ptr()
    return p


class _LpipsFunction(torch.autograd.Function):
    """(in0, in1 [N,3,H,W], module, save) -> distance [N], with nfi_lpips_backward as the backward
    (save 1 / 2: keep the workspace it reads for in0's gradient / for both)."""

    @staticmethod
    def forward(ctx, in0, in1, m, save):
        if not (in0.is_cuda and in1.is_cuda):
            raise _lib.NfiError('FusedLPIPS only runs on CUDA tensors (there is no CPU path)')
        ws = m.weights()
        if any(w.requires_grad for w in ws):
            raise _lib.NfiError('FusedLPIPS has no weight gradients; a weight requires grad')
        if in0.dim() != 4 or in0.shape[1] != 3 or in1.shape != in0.shape:
            raise _lib.NfiError('FusedLPIPS: in0 and in1 must both be [N,3,H,W], got %s and %s'
                                % (tuple(in0.shape), tuple(in1.shape)))
        N, _, H, W = in0.shape
        if N == 0 or H % 16 or W % 16 or H == 0 or W == 0:
            raise _lib.NfiError('FusedLPIPS: N > 0 and H, W multiples of 16 (four 2x2 pools), got %s'
                                % (tuple(in0.shape),))
        dev = in0.device
        if any(w.device != dev for w in ws) or in1.device != dev:
            raise _lib.NfiError('FusedLPIPS: weights and images on different devices')
        lib = _lib.load()
        with torch.cuda.device(dev):
            a = in0.detach().to(torch.float32).contiguous()
            b = in1.detach().to(torch.float32).contiguous()
            out = torch.empty(N, device=dev)
            p = _params(m, a, b, out, save)
            nbytes = lib.nfi_lpips_workspace_bytes(ctypes.byref(p))
            if nbytes == 0:
                _lib.check(1)
            work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            p.workspace, p.workspace_bytes = work.data_ptr(), nbytes
            stream = _lib.stream(dev)
            _lib.check(lib.nfi_lpips_forward(ctypes.byref(p), stream))
        # the backward reads the workspace and the tensors behind p's pointers
        ctx.state = (p, a, b, work, ws) if save else None
        ctx.in0_dtype, ctx.in1_dtype = in0.dtype, in1.dtype
        return out.to(in0.dtype)

    @staticmethod
    def backward(ctx, g_out):
        p, a, b, work, ws = _lib.take_saved(ctx, 'LPIPS')
        dev = a.device
        with torch.cuda.device(dev):
            g = g_out.to(torch.float32).contiguous()
            grad0 = torch.zeros_like(a)
            grad1 = torch.zeros_like(b) if p.save == 2 else None
            _lib.check(_lib.load().nfi_lpips_backward(ctypes.byref(p), _lib.ptr(g), _lib.ptr(grad0),
                                                      _lib.ptr(grad1), _lib.stream(dev)))
        del p, a, b, work, ws
        n0, n1 = ctx.needs_input_grad[:2]
        return (grad0.to(ctx.in0_dtype) if n0 else None,
                grad1.to(ctx.in1_dtype) if (n1 and grad1 is not None) else None, None, None)


def saved_preactivations(dist):
    """Every conv's pre-activation u kept by the saved forward behind ``dist`` (a FusedLPIPS output
    that requires grad, before its backward has run), as fp32 [2N,C,h,w] tensors (in0's images
    first) in layer order conv1_1 .. conv5_3.  Tests read the kernel's ReLU and pool branches from
    them."""
    p, a = _lib.find_saved(dist, 'LPIPS')[:2]
    lib = _lib.load()
    dev = a.device
    out = []
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)
        level = 0
        for i, (_, cout) in enumerate(CONV_CHANNELS):
            if i in (2, 4, 7, 10):
                level += 1
            u = torch.empty(2 * p.n, p.height >> level, p.width >> level, cout, device=dev)
            _lib.check(lib.nfi_lpips_saved_preactivation(ctypes.byref(p), i, _lib.ptr(u), stream))
            out.append(u.permute(0, 3, 1, 2))
    return out
