"""The synthesis network's parameter backward restated in float64 in the decomposition the sm_90a
kernels use (csrc/nfi_synth.cu, run_backward with parameter gradients), one modulated layer at a
time:

    g     = dy lrelu'(u) sqrt(2)                     (act_backward_kernel: bias and noise sums)
    dacc  = g d,  dd_part = sum_pos g (acc d)
    dW    = sum_{b,p} dacc[p + a(tap)] x~[p + x(tap)]   (wgrad_tc_kernel, x~ = x s)
          - W sum_b dd_part d^2 s^2                   (wgrad_reduce_kernel, demodulation term)

with the up layer's GEMM reading the four parity phases of the FIR adjoint's raw gradient:
raw (2i+ky, 2j+kx) = phase (ky%2, kx%2) at (i + ky//2, j + kx//2), against x~ on the
low-resolution grid.  ToRGB is the same GEMM with one tap, no demodulation, dimg for dacc.
The affine and b4.const gradients follow the data gradient ds of tests/synthesis_backward_oracle.py
through styles = (A w / sqrt(w_dim) + b) gain."""
import math

import torch
import torch.nn.functional as F

from oracle import synthesis_oracle as SO


def layer_param_grads(p, prefix, x, w, noise, up, dy):
    """-> dict of weight / bias / affine.weight / affine.bias / noise / x gradients of
    ``SO.synthesis_layer(p, prefix, x, w, noise, up, f)`` for the upstream gradient ``dy``."""
    f = SO.fir_kernel(x.device, x.dtype)
    W = p[prefix + '.weight']
    A, ab = p[prefix + '.affine.weight'], p[prefix + '.affine.bias']
    D = A.shape[1]
    s = w @ A.t() / math.sqrt(D) + ab                           # [B, cin]
    xs = x * s[:, :, None, None]                                # x~
    B, cout = x.shape[0], W.shape[0]
    if up:
        raw = F.conv_transpose2d(xs, W.transpose(0, 1), stride=2)
        acc = F.conv2d(raw.reshape(B * cout, 1, *raw.shape[2:]), (f * 4)[None, None], padding=1)
        acc = acc.view(B, cout, *acc.shape[2:])
    else:
        acc = F.conv2d(xs, W, padding=1)
    d = (s[:, None, :] ** 2 * W.square().sum(dim=(2, 3))[None]).sum(-1).add(1e-8).rsqrt()  # [B, cout]
    out = acc * d[:, :, None, None]
    if noise is not None:
        out = out + noise
    u = (out + p[prefix + '.bias'].view(1, -1, 1, 1)) * math.sqrt(2)
    g = dy * ((u > 0).to(dy.dtype) * 0.8 + 0.2) * math.sqrt(2)
    dacc = g * d[:, :, None, None]
    dd_part = (g * acc * d[:, :, None, None]).sum(dim=(2, 3))  # [B, cout]
    demod = torch.einsum('bo,bi->oi', dd_part * d ** 2, s ** 2)
    dW = torch.zeros_like(W)
    if up:
        h = x.shape[2]
        draw = F.conv_transpose2d(dacc.reshape(B * cout, 1, *dacc.shape[2:]), (f * 4)[None, None],
                                  padding=1).view(B, cout, 2 * h + 1, 2 * h + 1)
        phases = [[draw[:, :, py::2, px::2] for px in range(2)] for py in range(2)]
        for ky in range(3):
            for kx in range(3):
                ph = phases[ky % 2][kx % 2][:, :, ky // 2:ky // 2 + h, kx // 2:kx // 2 + h]
                dW[:, :, ky, kx] = torch.einsum('bohw,bihw->oi', ph, xs)
    else:
        H, Wd = x.shape[2], x.shape[3]
        xp = F.pad(xs, (1, 1, 1, 1))
        for ky in range(3):
            for kx in range(3):
                dW[:, :, ky, kx] = torch.einsum('bohw,bihw->oi', dacc, xp[:, :, ky:ky + H, kx:kx + Wd])
    dW = dW - W * demod[:, :, None, None]
    # the style gradient through the data path (the transpose of the conv) and demodulation
    ds = _style_grad(xs, x, s, W, dacc, dd_part, d, up, f)
    return {
        'weight': dW,
        'bias': g.sum(dim=(0, 2, 3)),
        'noise': g.sum(dim=1, keepdim=True),
        'affine.weight': ds.t() @ w / math.sqrt(D),
        'affine.bias': ds.sum(0),
    }


def _style_grad(xs, x, s, W, dacc, dd_part, d, up, f):
    """ds[b,ci] = sum_p dx~ x  -  s sum_o dd_part d^2 wsq[o,ci]  (dcoef_backward_kernel)."""
    xs = xs.detach().requires_grad_()
    if up:
        B, cout = xs.shape[0], W.shape[0]
        raw = F.conv_transpose2d(xs, W.transpose(0, 1), stride=2)
        a = F.conv2d(raw.reshape(B * cout, 1, *raw.shape[2:]), (f * 4)[None, None], padding=1)
        a = a.view(B, cout, *a.shape[2:])
    else:
        a = F.conv2d(xs, W, padding=1)
    (dxs,) = torch.autograd.grad(a, xs, dacc)
    wsq = W.square().sum(dim=(2, 3))
    return (dxs * x).sum(dim=(2, 3)) - s * ((dd_part * d ** 2) @ wsq)


def torgb_param_grads(p, prefix, x, w, dimg):
    """ToRGB: x~ = x s / sqrt(cin), one tap, no demodulation."""
    W = p[prefix + '.weight']
    A, ab = p[prefix + '.affine.weight'], p[prefix + '.affine.bias']
    D, cin = A.shape[1], W.shape[1]
    s = (w @ A.t() / math.sqrt(D) + ab) / math.sqrt(cin)
    xs = x * s[:, :, None, None]
    dW = torch.einsum('bohw,bihw->oi', dimg, xs)[:, :, None, None]
    dxs = torch.einsum('bohw,oi->bihw', dimg, W[:, :, 0, 0])
    ds = (dxs * x).sum(dim=(2, 3)) / math.sqrt(cin)
    return {'weight': dW, 'bias': dimg.sum(dim=(0, 2, 3)),
            'affine.weight': ds.t() @ w / math.sqrt(D), 'affine.bias': ds.sum(0)}
