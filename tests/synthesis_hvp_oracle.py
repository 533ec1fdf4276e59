"""The path-length regulariser's double backward restated in float64 in the decomposition the
sm_90a kernels use (csrc/nfi_synth.cu, run_hvp) -- TEST INFRASTRUCTURE.

With n the planes cotangent and t the cotangent of g_ws = J_ws^T n, the gradient of
Phi = <t, J_ws^T n> with respect to ws, every parameter and the noise tensors is the tangent, along
ws + eps t, of the first-order backward with cotangent n.  Notation as in
tests/synthesis_param_backward_oracle.py; a trailing ``_t`` is the tangent.  Per modulated layer:

tangent forward:
    s_t   = A t / sqrt(D)                        d_t  = -d^3 sum_i wsq s s_t
    x~_t  = x_t s + x s_t                        acc_t = conv(x~_t, W)
    u_t   = sqrt(2) (acc_t d + acc d_t)          v_t  = lrelu'(u) u_t
backward beside its tangent, given dv and dv_t (the gradient of v and its tangent):
    g_t    = dv_t lrelu'(u) sqrt(2)              (lrelu'' = 0)
    dacc_t = g_t d + g d_t                       dd_t = sum_p g_t (acc d) + g u_t / sqrt(2)
    dx~_t  = conv^T(dacc_t, W)
    ds_t   = sum_p dx~_t x + dx~ x_t - s_t sum_o dd d^2 wsq - s sum_o (dd_t d^2 + 2 dd d d_t) wsq
    dx_t   = dx~_t s + dx~ s_t                   (-> the previous layer's dv_t)
outputs:
    weight  sum dacc_t (x) x~ + dacc (x) x~_t - W sum_b [dd_t d^2 s^2 + 2 dd d d_t s^2 + 2 dd d^2 s s_t]
    bias    sum g_t       noise  sum_c g_t
    affine  (ds_t^T w + ds^T t) gain / sqrt(D),  sum_b ds_t gain
    ws      ds_t A gain / sqrt(D)
ToRGB: dimg does not depend on ws, so dx~_rgb_t = 0, ds_rgb_t = sum_p dx~_rgb x_t, weight
sum dimg (x) x~_t, bias 0.  b4.const: x_t = 0, const gradient sum_b dx~_t s + dx~ s_t.
"""
import math

import torch
import torch.nn.functional as F

from oracle.synthesis_oracle import fir_kernel

SQRT2 = math.sqrt(2)


def _lrelu_grad(u):
    return torch.where(u > 0, torch.ones_like(u), torch.full_like(u, 0.2))


def _conv(xs, W, up, f):
    if up:
        B, cout = xs.shape[0], W.shape[0]
        raw = F.conv_transpose2d(xs, W.transpose(0, 1), stride=2)
        acc = F.conv2d(raw.reshape(B * cout, 1, *raw.shape[2:]), (f * 4)[None, None], padding=1)
        return acc.view(B, cout, *acc.shape[2:])
    return F.conv2d(xs, W, padding=1)


def _conv_t(dacc, xs, W, up, f):
    """conv^T(dacc, W): the adjoint of the (linear) convolution at xs's shape."""
    xs = torch.zeros_like(xs).requires_grad_()
    (dx,) = torch.autograd.grad(_conv(xs, W, up, f), xs, dacc)
    return dx


def _wgrad(dacc, xs, W, up, f):
    """sum_{b,p} dacc (x) xs over the taps: the conv's weight gradient without demodulation."""
    W = W.detach().clone().requires_grad_()
    (dW,) = torch.autograd.grad(_conv(xs, W, up, f), W, dacc)
    return dW


def layer_forward(p, prefix, x, x_t, w, t, noise, up, f):
    """One modulated layer and its tangent; x_t None = an input that does not depend on ws."""
    W = p[prefix + '.weight']
    A, ab = p[prefix + '.affine.weight'], p[prefix + '.affine.bias']
    D = A.shape[1]
    s = w @ A.t() / math.sqrt(D) + ab
    s_t = t @ A.t() / math.sqrt(D)
    wsq = W.square().sum(dim=(2, 3))
    d = (s.square() @ wsq.t() + 1e-8).rsqrt()
    d_t = -d ** 3 * ((s * s_t) @ wsq.t())
    if x_t is None:
        x_t = torch.zeros_like(x)
    xs = x * s[:, :, None, None]
    xs_t = x_t * s[:, :, None, None] + x * s_t[:, :, None, None]
    acc = _conv(xs, W, up, f)
    acc_t = _conv(xs_t, W, up, f)
    u = acc * d[:, :, None, None]
    if noise is not None:
        u = u + noise
    u = (u + p[prefix + '.bias'].view(1, -1, 1, 1)) * SQRT2
    u_t = SQRT2 * (acc_t * d[:, :, None, None] + acc * d_t[:, :, None, None])
    v = F.leaky_relu(u, 0.2)
    v_t = _lrelu_grad(u) * u_t
    L = dict(W=W, A=A, D=D, s=s, s_t=s_t, wsq=wsq, d=d, d_t=d_t, x=x, x_t=x_t, xs=xs, xs_t=xs_t,
             acc=acc, u=u, u_t=u_t, up=up, w=w, t=t)
    return L, v, v_t


def layer_backward(L, dv, dv_t, f):
    """-> (dx~, dx~_t, dict of the tangents of the layer's gradients: weight, bias, noise,
    affine.weight, affine.bias, ws (the row's HVP part))."""
    s, s_t, d, d_t, wsq = L['s'], L['s_t'], L['d'], L['d_t'], L['wsq']
    lg = _lrelu_grad(L['u'])
    g = dv * lg * SQRT2
    g_t = dv_t * lg * SQRT2
    dd = (g * L['acc'] * d[:, :, None, None]).sum(dim=(2, 3))
    dd_t = (g_t * L['acc'] * d[:, :, None, None] + g * L['u_t'] / SQRT2).sum(dim=(2, 3))
    dacc = g * d[:, :, None, None]
    dacc_t = g_t * d[:, :, None, None] + g * d_t[:, :, None, None]
    dxs = _conv_t(dacc, L['xs'], L['W'], L['up'], f)
    dxs_t = _conv_t(dacc_t, L['xs'], L['W'], L['up'], f)
    P = (dd * d ** 2) @ wsq
    Q = (dd_t * d ** 2 + 2 * dd * d * d_t) @ wsq
    ds = (dxs * L['x']).sum(dim=(2, 3)) - s * P
    ds_t = (dxs_t * L['x'] + dxs * L['x_t']).sum(dim=(2, 3)) - s_t * P - s * Q
    dem_t = (torch.einsum('bo,bi->oi', dd_t * d ** 2 + 2 * dd * d * d_t, s ** 2)
             + torch.einsum('bo,bi->oi', 2 * dd * d ** 2, s * s_t))
    W = L['W']
    dW_t = (_wgrad(dacc_t, L['xs'], W, L['up'], f) + _wgrad(dacc, L['xs_t'], W, L['up'], f)
            - W * dem_t[:, :, None, None])
    scale = 1 / math.sqrt(L['D'])
    out = {'weight': dW_t, 'bias': g_t.sum(dim=(0, 2, 3)), 'noise': g_t.sum(dim=1, keepdim=True),
           'affine.weight': (ds_t.t() @ L['w'] + ds.t() @ L['t']) * scale,
           'affine.bias': ds_t.sum(0), 'ws': ds_t @ L['A'] * scale}
    return dxs, dxs_t, out


def torgb_hvp(p, prefix, x, x_t, w, t, dimg):
    """ToRGB with the constant cotangent dimg -> (dx~, dict of gradient tangents)."""
    W = p[prefix + '.weight']
    A, ab = p[prefix + '.affine.weight'], p[prefix + '.affine.bias']
    D, cin = A.shape[1], W.shape[1]
    gain = 1 / math.sqrt(cin)
    s = (w @ A.t() / math.sqrt(D) + ab) * gain
    s_t = t @ A.t() / math.sqrt(D) * gain
    xs_t = x_t * s[:, :, None, None] + x * s_t[:, :, None, None]
    dxs = torch.einsum('bohw,oi->bihw', dimg, W[:, :, 0, 0])
    ds = (dxs * x).sum(dim=(2, 3))
    ds_t = (dxs * x_t).sum(dim=(2, 3))
    scale = gain / math.sqrt(D)
    out = {'weight': torch.einsum('bohw,bihw->oi', dimg, xs_t)[:, :, None, None],
           'bias': torch.zeros_like(p[prefix + '.bias']),
           'affine.weight': (ds_t.t() @ w + ds.t() @ t) * scale,
           'affine.bias': ds_t.sum(0) * gain, 'ws': ds_t @ A * scale}
    return dxs, s, s_t, out


def synthesis_hvp(p, ws, noises, n_img, t_ws):
    """-> (g_ws [B,num_ws,w_dim], {parameter name: gradient}, {noise key: gradient}) of
    Phi = <t_ws, J_ws^T n_img> for ``oracle.synthesis_oracle.synthesis_forward(p, ws, noises)``
    (n_img channel-first [B,96,R,R], as the reference)."""
    meta = p['meta']
    f = fir_kernel(ws.device, ws.dtype)
    noises = noises or {}
    blocks, x, x_t, w_idx = [], None, None, 0
    for r in meta['resolutions']:
        pre = 'b%d' % r
        blk = dict(pre=pre)
        if r == 4:
            x = p[pre + '.const'].unsqueeze(0).repeat(ws.shape[0], 1, 1, 1)
            x_t, n_conv = None, 1
        else:
            blk['conv0'], x, x_t = layer_forward(p, pre + '.conv0', x, x_t, ws[:, w_idx],
                                                 t_ws[:, w_idx], noises.get(pre + '.conv0'), True, f)
            blk['row0'], n_conv = w_idx, 2
        blk['conv1'], x, x_t = layer_forward(p, pre + '.conv1', x, x_t, ws[:, w_idx + n_conv - 1],
                                             t_ws[:, w_idx + n_conv - 1], noises.get(pre + '.conv1'),
                                             False, f)
        blk['row1'], blk['row_rgb'] = w_idx + n_conv - 1, w_idx + n_conv
        blk['v'], blk['v_t'] = x, x_t
        blocks.append(blk)
        w_idx += n_conv
    g_ws = torch.zeros_like(ws)
    grads, g_noise = {}, {}
    dimg, nxt = n_img, None   # nxt: (dx~, dx~_t, s, s_t) of conv0 of the block above
    for i in reversed(range(len(blocks))):
        blk, pre = blocks[i], blocks[i]['pre']
        row = blk['row_rgb']
        dxr, s_r, s_rt, out = torgb_hvp(p, pre + '.torgb', blk['v'], blk['v_t'], ws[:, row],
                                        t_ws[:, row], dimg)
        g_ws[:, row] += out.pop('ws')
        grads.update({pre + '.torgb.' + k: v for k, v in out.items()})
        dv = dxr * s_r[:, :, None, None]
        dv_t = dxr * s_rt[:, :, None, None]
        if nxt is not None:
            dxs, dxs_t, s, s_t = nxt
            dv = dv + dxs * s[:, :, None, None]
            dv_t = dv_t + dxs_t * s[:, :, None, None] + dxs * s_t[:, :, None, None]
        if i:
            B, C, H, W = dimg.shape
            dimg = F.conv2d(dimg.reshape(B * C, 1, H, W), (f * 4)[None, None], stride=2,
                            padding=1).view(B, C, H // 2, W // 2)
        L1 = blk['conv1']
        dxs, dxs_t, out = layer_backward(L1, dv, dv_t, f)
        g_ws[:, blk['row1']] += out.pop('ws')
        if pre + '.conv1' in noises:
            g_noise[pre + '.conv1'] = out['noise']
        out.pop('noise')
        grads.update({pre + '.conv1.' + k: v for k, v in out.items()})
        if i == 0:
            s, s_t = L1['s'], L1['s_t']
            grads[pre + '.const'] = (dxs_t * s[:, :, None, None]
                                     + dxs * s_t[:, :, None, None]).sum(0)
            break
        dv = dxs * L1['s'][:, :, None, None]
        dv_t = dxs_t * L1['s'][:, :, None, None] + dxs * L1['s_t'][:, :, None, None]
        L0 = blk['conv0']
        dxs, dxs_t, out = layer_backward(L0, dv, dv_t, f)
        g_ws[:, blk['row0']] += out.pop('ws')
        if pre + '.conv0' in noises:
            g_noise[pre + '.conv0'] = out['noise']
        out.pop('noise')
        grads.update({pre + '.conv0.' + k: v for k, v in out.items()})
        nxt = (dxs, dxs_t, L0['s'], L0['s_t'])
    return g_ws, grads, g_noise
