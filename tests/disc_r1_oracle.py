"""The R1 regulariser's double backward of the discriminator backbone, restated in float64 as the
decomposition nfi_disc_backward_hvp runs (include/nfi_disc_r1.h) -- TEST INFRASTRUCTURE.

With L = sum_b g_logits[b] logits[b] and a tangent t of the image, ``r1(p, img, cmap, g_logits, t)``
returns the gradients of Phi = <t, dL/dimg> with respect to every parameter (by state_dict name, as
oracle/disc_oracle.py takes them), the image, cmap and g_logits, computed as:

- a tangent forward along t on fixed leaky-ReLU branches (lrelu'' = 0): every layer but the
  minibatch std is its linear map times lrelu';
- the first-order cotangents g of the 4x4 epilogue, whose tangents are zero (they do not depend on
  the image), so the epilogue's weight terms are g (x) a-dot only and its biases get zero;
- the minibatch std's second-order term, which seeds g-dot of the last block's output;
- the blocks' reverse walk of [g; g-dot] through the same linear maps, each weight's gradient
  sum g-dot (x) a + g (x) a-dot and each bias's sum g-dot.

``branches`` (keyed as nerf_from_image_b200.discriminator.saved_preactivations, channel-last where
that is) fixes the branches; by default each layer's own pre-activation's sign does.
"""
import math

import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from oracle import disc_oracle as DO

S2 = math.sqrt(2)
EPS = 1e-8


def _mask(u, branch):
    b = branch if branch is not None else u
    return torch.where(b > 0, torch.ones_like(u), torch.full_like(u, 0.2))


def _fir_k(x):
    C = x.shape[1]
    return DO.fir(x.dtype, x.device)[None, None].expand(C, 1, 4, 4).contiguous()


def down(x):       # downsample2d: the FIR, stride 2, pad 1
    return F.conv2d(x, _fir_k(x), padding=1, stride=2, groups=x.shape[1])


def down_adjoint(g, shape):
    return conv2d_input(shape, _fir_k(g), g, stride=2, padding=1, groups=g.shape[1])


def up(a):         # filter2d^T: [B,C,r,r] -> [B,C,r+1,r+1]
    return F.conv_transpose2d(a, _fir_k(a), padding=1, groups=a.shape[1])


def up_adjoint(g):
    return F.conv2d(g, _fir_k(g), padding=1, groups=g.shape[1])


# ---- minibatch std (groups of 4: images j, j + B/4, j + B/2, j + 3B/4)
def _groups(x):
    return x.reshape(4, -1, *x.shape[1:])


def mbstd(x):
    """sd [B/4] and xs [B,513,4,4]."""
    v = _groups(x)
    m = v.mean(0)
    s = ((v - m).square().mean(0) + EPS).sqrt()
    sd = s.flatten(1).mean(1)
    return sd, torch.cat([x, sd.repeat(4)[:, None, None, None].expand(-1, 1, 4, 4)], 1)


def mbstd_tangent(x, dx):
    """sd-dot [B/4] and xs-dot [B,513,4,4] along x-dot."""
    v, dv = _groups(x), _groups(dx)
    c, dc = v - v.mean(0), dv - dv.mean(0)
    s = (c.square().mean(0) + EPS).sqrt()
    dsd = ((c * dc).sum(0) / (4 * s)).flatten(1).mean(1)
    return dsd, torch.cat([dx, dsd.repeat(4)[:, None, None, None].expand(-1, 1, 4, 4)], 1)


def mbstd_backward(gxs, x):
    """g_x [B,512,4,4] of the std layer, from g_xs [B,513,4,4]."""
    v = _groups(x)
    c = v - v.mean(0)
    s = (c.square().mean(0) + EPS).sqrt()
    G = _groups(gxs[:, 512]).sum(dim=(0, 2, 3))     # [B/4]
    k = (G / (16 * 512))[:, None, None, None]
    return gxs[:, :512] + (k * c / (4 * s)).reshape(x.shape)


def mbstd_hvp(gxs, x, dx):
    """g-dot_x: the tangent of mbstd_backward along x-dot with g_xs fixed."""
    v, dv = _groups(x), _groups(dx)
    c, dc = v - v.mean(0), dv - dv.mean(0)
    s = (c.square().mean(0) + EPS).sqrt()
    ds = (c * dc).sum(0) / (4 * s)
    G = _groups(gxs[:, 512]).sum(dim=(0, 2, 3))
    k = (G / (16 * 512 * 4))[:, None, None, None]
    return (k * (dc / s - c * ds / s.square())).reshape(x.shape)


# ---- the 4x4 epilogue
def epilogue_forward(p, x4, cmap, br=None):
    br = br or {}
    sd, xs = mbstd(x4)
    wc = p['b4.conv.weight'] / math.sqrt(513 * 9)
    u4 = (F.conv2d(xs, wc, padding=1) + p['b4.conv.bias'].view(1, -1, 1, 1)) * S2
    m4 = _mask(u4, br.get('b4.conv'))
    a4 = u4 * m4
    uf = (a4.flatten(1) @ (p['b4.fc.weight'] / math.sqrt(8192)).T + p['b4.fc.bias']) * S2
    mf = _mask(uf, br.get('b4.fc'))
    hf = uf * mf
    out = hf @ (p['b4.out.weight'] / math.sqrt(512)).T + p['b4.out.bias']
    lg = (out * cmap).sum(1, keepdim=True) / math.sqrt(cmap.shape[1]) if cmap is not None else out
    return dict(xs=xs, m4=m4, a4=a4, mf=mf, hf=hf, out=out, logits=lg)


def epilogue_r1(p, x4, cmap, g_logits, dx4, br=None):
    """The epilogue's part: gradients of the epilogue parameters, cmap and g_logits, and [g; g-dot]
    of x4."""
    f = epilogue_forward(p, x4, cmap, br)
    wc = p['b4.conv.weight'] / math.sqrt(513 * 9)
    wf = p['b4.fc.weight'] / math.sqrt(8192)
    wo = p['b4.out.weight'] / math.sqrt(512)
    N = cmap.shape[1] if cmap is not None else 1
    # tangent forward
    _, dxs = mbstd_tangent(x4, dx4)
    da4 = f['m4'] * S2 * F.conv2d(dxs, wc, padding=1)
    dhf = f['mf'] * S2 * (da4.flatten(1) @ wf.T)
    dout = dhf @ wo.T
    dlg = (dout * cmap).sum(1, keepdim=True) / math.sqrt(N) if cmap is not None else dout
    # first-order cotangents (their tangents are zero)
    gl = g_logits.reshape(-1, 1)
    g_out = gl * cmap / math.sqrt(N) if cmap is not None else gl
    g_uf = f['mf'] * S2 * (g_out @ wo)
    g_u4 = (f['m4'] * S2 * (g_uf @ wf).reshape(f['a4'].shape))
    g_xs = conv2d_input(f['xs'].shape, wc, g_u4, padding=1)
    res = {
        'b4.out.weight': g_out.T @ dhf / math.sqrt(512),
        'b4.out.bias': torch.zeros_like(p['b4.out.bias']),
        'b4.fc.weight': g_uf.T @ da4.flatten(1) / math.sqrt(8192),
        'b4.fc.bias': torch.zeros_like(p['b4.fc.bias']),
        'b4.conv.weight': conv2d_weight(dxs, wc.shape, g_u4, padding=1) / math.sqrt(513 * 9),
        'b4.conv.bias': torch.zeros_like(p['b4.conv.bias']),
        'g_logits': dlg.reshape(g_logits.shape),
    }
    if cmap is not None:
        res['cmap'] = gl * dout / math.sqrt(N)
    return res, mbstd_backward(g_xs, x4), mbstd_hvp(g_xs, x4, dx4), f


# ---- one resolution block (x [B,C,r,r] -> y [B,C',r/2,r/2])
def block_forward(p, k, x, br=None, r=None):
    br = br or {}
    c = x.shape[1]
    d = down(x)
    ws = p[k + 'skip.weight'] / math.sqrt(c)
    w0 = p[k + 'conv0.weight'] / math.sqrt(9 * c)
    w1 = p[k + 'conv1.weight'] / math.sqrt(9 * c)
    u0 = (F.conv2d(x, w0, padding=1) + p[k + 'conv0.bias'].view(1, -1, 1, 1)) * S2
    ma = _mask(u0, DO._cl(br.get(('conv0', r))))
    a = u0 * ma
    f = up(a)
    u1 = F.conv2d(f, w1, stride=2) + p[k + 'conv1.bias'].view(1, -1, 1, 1)
    m1 = _mask(u1, DO._cl(br.get(('conv1', r))))
    y = F.conv2d(d, ws) * (S2 / 2) + u1 * m1
    return dict(x=x, d=d, ma=ma, f=f, m1=m1, y=y, w0=w0, w1=w1, ws=ws)


def block_tangent(s, dx):
    da = s['ma'] * S2 * F.conv2d(dx, s['w0'], padding=1)
    df = up(da)
    dd = down(dx)
    dy = s['m1'] * F.conv2d(df, s['w1'], stride=2) + F.conv2d(dd, s['ws']) * (S2 / 2)
    return dict(dx=dx, df=df, dd=dd, dy=dy)


def block_r1(s, t, k, g_y, dg_y):
    """[g; g-dot] of the block's input and the R1 gradients of its parameters."""
    c = s['x'].shape[1]
    g_u1, dg_u1 = s['m1'] * g_y, s['m1'] * dg_y
    res = {
        k + 'conv1.bias': dg_u1.sum(dim=(0, 2, 3)),
        k + 'conv1.weight': (conv2d_weight(s['f'], s['w1'].shape, dg_u1, stride=2)
                             + conv2d_weight(t['df'], s['w1'].shape, g_u1, stride=2)) / math.sqrt(9 * c),
        k + 'skip.weight': (conv2d_weight(s['d'], s['ws'].shape, dg_y)
                            + conv2d_weight(t['dd'], s['ws'].shape, g_y)) * (S2 / 2) / math.sqrt(c),
    }
    out = []
    for g, dg in ((g_u1, g_y), (dg_u1, dg_y)):
        g_a = up_adjoint(conv2d_input(s['f'].shape, s['w1'], g, stride=2))
        g_u0 = s['ma'] * S2 * g_a
        g_d = conv2d_input(s['d'].shape, s['ws'], dg) * (S2 / 2)
        out.append((g_u0, conv2d_input(s['x'].shape, s['w0'], g_u0, padding=1) + down_adjoint(g_d, s['x'].shape)))
    (g_u0, g_x), (dg_u0, dg_x) = out
    res[k + 'conv0.bias'] = dg_u0.sum(dim=(0, 2, 3))
    res[k + 'conv0.weight'] = (conv2d_weight(s['x'], s['w0'].shape, dg_u0, padding=1)
                               + conv2d_weight(t['dx'], s['w0'].shape, g_u0, padding=1)) / math.sqrt(9 * c)
    return res, g_x, dg_x


# ---- the whole backbone
def r1(p, img, cmap, g_logits, t, branches=None):
    br = branches or {}
    R, nc = img.shape[2], img.shape[1]
    rs = DO.block_resolutions(R)
    k0 = 'b%d.' % R
    wr = p[k0 + 'fromrgb.weight'] / math.sqrt(nc)
    u = (F.conv2d(img, wr) + p[k0 + 'fromrgb.bias'].view(1, -1, 1, 1)) * S2
    m0 = _mask(u, DO._cl(br.get('fromrgb')))
    x = u * m0
    dx = m0 * S2 * F.conv2d(t, wr)
    saved = []
    for r in rs:
        s = block_forward(p, 'b%d.' % r, x, br, r)
        tg = block_tangent(s, dx)
        saved.append((r, s, tg))
        x, dx = s['y'], tg['dy']
    res, g, dg, _ = epilogue_r1(p, x, cmap, g_logits, dx, br)
    for r, s, tg in reversed(saved):
        rb, g, dg = block_r1(s, tg, 'b%d.' % r, g, dg)
        res.update(rb)
    g_u, dg_u = m0 * S2 * g, m0 * S2 * dg
    res[k0 + 'fromrgb.bias'] = dg_u.sum(dim=(0, 2, 3))
    res[k0 + 'fromrgb.weight'] = (conv2d_weight(img, wr.shape, dg_u)
                                  + conv2d_weight(t, wr.shape, g_u)) / math.sqrt(nc)
    res['img'] = conv2d_input(img.shape, wr, dg_u)
    return res


def double_backward(p, img, cmap, g_logits, t, branches=None):
    """The same gradients by torch's float64 double backward through oracle/disc_oracle.py."""
    pd = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
    x = img.detach().clone().requires_grad_()
    c = cmap.detach().clone().requires_grad_() if cmap is not None else None
    gl = g_logits.detach().clone().reshape(-1, 1).requires_grad_()
    out = DO.backbone(pd, x, c, branches)
    gx, = torch.autograd.grad((out * gl).sum(), x, create_graph=True)
    (gx * t).sum().backward()
    res = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in pd.items()}
    res['img'] = x.grad
    res['g_logits'] = gl.grad.reshape(g_logits.shape)
    if c is not None:
        res['cmap'] = c.grad
    return res
