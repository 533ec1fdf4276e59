"""The synthesis network's backward to the latents, restated in the decomposition of the sm_90a
kernels (``csrc/nfi_synth.cu``, ``run_backward``) -- TEST INFRASTRUCTURE.

``synthesis_backward(p, ws, noises, g_img)`` returns dL/dws for ``L = <g_img,
oracle.synthesis_oracle.synthesis_forward(p, ws, noises)>`` with every parameter frozen, computed
the way the kernels compute it rather than by autograd:

per layer (s = affine(w), x~ = x s, acc = conv(x~, W), d = rsqrt(sum_i wsq[o,i] s_i^2 + 1e-8),
u = (acc d + noise + bias) sqrt(2), v = lrelu(u)), given the gradient dv of v:
    g     = dv lrelu'(u) sqrt(2)          dacc = g d           dd[b,o] = sum_pos g acc
    dx~   = conv^T(dacc, W)               dx = dx~ s           (-> the previous layer's dv)
    ds[i] = sum_pos dx~ x  -  s_i sum_o dd_o d_o^3 wsq[o,i]
    dws[b, row] += gain / sqrt(w_dim) * ds @ A
The up layer's adjoint is the FIR's (a correlation with the same symmetric taps) into the
(2H+1)^2 raw gradient, split into its four parity phases; tap (ky,kx) then reads phase
(ky%2, kx%2) shifted by (ky//2, kx//2): nine stride-1 taps.  ToRGB: g = Wrgb^T dimg, dv += g s_rgb,
ds_rgb = sum_pos g v (gain 1/sqrt(Cin)); the running image's gradient goes one block down through
the adjoint of ``upsample_img``.  ToRGB of block i and conv0 of block i+1 share a ``ws`` row.
"""
import math

import torch
import torch.nn.functional as F

from oracle.synthesis_oracle import affine, fir_kernel


def _lrelu_grad(u):
    return torch.where(u > 0, torch.ones_like(u), torch.full_like(u, 0.2))


def _layer_forward(p, prefix, x, w, noise, up, f):
    """The forward of one SynthesisLayer, keeping what the backward reads."""
    W = p[prefix + '.weight']
    s = affine(p, prefix, w)
    wsq = W.square().sum(dim=[2, 3])                                     # [Cout, Cin]
    d = (s.square() @ wsq.t() + 1e-8).rsqrt()                            # [B, Cout]
    xs = x * s[:, :, None, None]
    if up:
        raw = F.conv_transpose2d(xs, W.transpose(0, 1), stride=2)       # [B, Cout, 2H+1, 2W+1]
        B, C = raw.shape[:2]
        acc = F.conv2d(raw.reshape(B * C, 1, *raw.shape[2:]), (f * 4)[None, None], padding=1)
        acc = acc.view(B, C, acc.shape[2], acc.shape[3])
    else:
        acc = F.conv2d(xs, W, padding=1)
    u = acc * d[:, :, None, None]
    if noise is not None:
        u = u + noise
    u = (u + p[prefix + '.bias'].view(1, -1, 1, 1)) * math.sqrt(2)
    return dict(x=x, s=s, wsq=wsq, d=d, acc=acc, u=u, W=W, up=up), F.leaky_relu(u, 0.2)


def _layer_backward(L, dv, f):
    """-> (dx~ (gradient of the styled input), ds)."""
    g = dv * _lrelu_grad(L['u']) * math.sqrt(2)
    dd = (g * L['acc']).sum(dim=[2, 3])                                  # [B, Cout]
    dacc = g * L['d'][:, :, None, None]
    W = L['W']
    if L['up']:
        B, C, OH, OW = dacc.shape
        # FIR adjoint: correlation with the (symmetric) taps over the zero-padded gradient
        raw = F.conv2d(F.pad(dacc.reshape(B * C, 1, OH, OW), (2, 2, 2, 2)), (f * 4)[None, None])
        raw = raw.view(B, C, OH + 1, OW + 1)
        h, w = OH // 2, OW // 2
        phases = torch.zeros(2, 2, B, C, h + 1, w + 1, dtype=raw.dtype, device=raw.device)
        for py in range(2):
            for px in range(2):
                ph = raw[:, :, py::2, px::2]
                phases[py, px, :, :, :ph.shape[2], :ph.shape[3]] = ph
        dx = 0
        for ky in range(3):
            for kx in range(3):
                a = phases[ky % 2, kx % 2, :, :, ky // 2:ky // 2 + h, kx // 2:kx // 2 + w]
                dx = dx + torch.einsum('bohw,oc->bchw', a, W[:, :, ky, kx])
    else:
        # stride 1, pad 1: the correlation with flipped taps and transposed channels
        dx = F.conv2d(dacc, W.transpose(0, 1).flip(2, 3), padding=1)
    ds = (dx * L['x']).sum(dim=[2, 3]) - L['s'] * ((dd * L['d'] ** 3) @ L['wsq'])
    return dx, ds


def _to_ws(p, prefix, ds, gain):
    A = p[prefix + '.affine.weight']
    return (ds @ A) * (gain / math.sqrt(A.shape[1]))


def synthesis_backward(p, ws, noises, g_img):
    """dL/dws [B, num_ws, w_dim] for the upstream gradient ``g_img`` [B, img_channels, R, R]
    of ``synthesis_forward(p, ws, noises)`` (channel-first, as the reference)."""
    meta = p['meta']
    f = fir_kernel(ws.device, ws.dtype)
    noises = noises or {}
    # ---- forward, keeping each layer's tensors
    blocks, x, w_idx = [], None, 0
    for r in meta['resolutions']:
        pre = 'b%d' % r
        blk = dict(pre=pre)
        if r == 4:
            x = p[pre + '.const'].unsqueeze(0).repeat(ws.shape[0], 1, 1, 1)
            n_conv = 1
        else:
            blk['conv0'], x = _layer_forward(p, pre + '.conv0', x, ws[:, w_idx],
                                             noises.get(pre + '.conv0'), True, f)
            blk['row0'] = w_idx
            n_conv = 2
        blk['conv1'], x = _layer_forward(p, pre + '.conv1', x, ws[:, w_idx + n_conv - 1],
                                         noises.get(pre + '.conv1'), False, f)
        blk['row1'] = w_idx + n_conv - 1
        wt = p[pre + '.torgb.weight']
        blk['s_rgb'] = affine(p, pre + '.torgb', ws[:, w_idx + n_conv]) / math.sqrt(wt.shape[1])
        blk['v'], blk['row_rgb'] = x, w_idx + n_conv
        blocks.append(blk)
        w_idx += n_conv
    # ---- backward, last block first
    g_ws = torch.zeros_like(ws)
    dimg, dx_next, s_next = g_img, None, None
    for i in reversed(range(len(blocks))):
        blk, pre = blocks[i], blocks[i]['pre']
        wt = p[pre + '.torgb.weight']
        g = torch.einsum('bnhw,nc->bchw', dimg, wt[:, :, 0, 0])          # Wrgb^T dimg
        dv = g * blk['s_rgb'][:, :, None, None]
        ds_rgb = (g * blk['v']).sum(dim=[2, 3])
        g_ws[:, blk['row_rgb']] += _to_ws(p, pre + '.torgb', ds_rgb, 1 / math.sqrt(wt.shape[1]))
        if dx_next is not None:                                          # conv0 of block i+1
            dv = dv + dx_next * s_next[:, :, None, None]
        if i:                                                            # upsample_img adjoint
            B, C, H, W = dimg.shape
            dimg = F.conv2d(dimg.reshape(B * C, 1, H, W), (f * 4)[None, None], stride=2,
                            padding=1).view(B, C, H // 2, W // 2)
        dx, ds = _layer_backward(blk['conv1'], dv, f)
        g_ws[:, blk['row1']] += _to_ws(p, pre + '.conv1', ds, 1.0)
        if i == 0:
            break
        L1 = blk['conv1']
        dx, ds = _layer_backward(blk['conv0'], dx * L1['s'][:, :, None, None], f)
        g_ws[:, blk['row0']] += _to_ws(p, pre + '.conv0', ds, 1.0)
        dx_next, s_next = dx, blk['conv0']['s']
    return g_ws
