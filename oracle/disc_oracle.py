"""A float64 restatement of the reference's DiscriminatorBackbone from the image and the
conditioning map on (models/stylegan.py:493-676) -- TEST INFRASTRUCTURE.

``backbone(p, img, cmap)`` takes the backbone's parameters by their state_dict names ('b128.conv0.
weight', 'b4.fc.bias', ...; the mapping network's are not read) and can take every leaky ReLU's
branch from ``branches`` (a dict keyed as ``nerf_from_image_b200.discriminator.saved_
preactivations``, channel-last where that is) instead of from its own pre-activation's sign.
"""
import math

import torch
import torch.nn.functional as F


def channels(r):
    return min(32768 // r, 512)


def block_resolutions(R):
    return [R >> i for i in range(int(math.log2(R)) - 2)]


def fir(dtype=torch.float64, device='cpu'):
    f = torch.tensor([1., 3., 3., 1.], dtype=dtype, device=device)
    f = f[:, None] * f[None, :]
    return f / f.sum()


def _lrelu(u, branch):
    pos = (branch > 0) if branch is not None else (u > 0)
    return torch.where(pos, u, 0.2 * u)


def _cl(t):   # channel-last [B,H,W,C] -> [B,C,H,W]
    return t.permute(0, 3, 1, 2) if t is not None else None


def _depthwise(x, f, stride, transpose):
    B, C, H, W = x.shape
    k = f[None, None].expand(C, 1, 4, 4)
    if transpose:
        return F.conv_transpose2d(x, k, padding=1, groups=C)
    return F.conv2d(x, k, padding=1, stride=stride, groups=C)


def backbone(p, img, cmap, branches=None):
    """Logits [B,1] of the backbone with parameters ``p`` on ``img`` [B,nc,R,R] and ``cmap``
    [B,cmap_dim] (None: unconditional)."""
    br = branches or {}
    R, nc = img.shape[2], img.shape[1]
    f = fir(img.dtype, img.device)
    x = None
    for i, r in enumerate(block_resolutions(R)):
        k = 'b%d.' % r
        if i == 0:
            w = p[k + 'fromrgb.weight'] / math.sqrt(nc)
            x = _lrelu((F.conv2d(img, w) + p[k + 'fromrgb.bias'].view(1, -1, 1, 1)) * math.sqrt(2),
                       _cl(br.get('fromrgb')))
        c = x.shape[1]
        ws = p[k + 'skip.weight'] / math.sqrt(c)
        y = F.conv2d(_depthwise(x, f, 2, False), ws) * (math.sqrt(2) / 2)
        w0 = p[k + 'conv0.weight'] / math.sqrt(9 * c)
        a = _lrelu((F.conv2d(x, w0, padding=1) + p[k + 'conv0.bias'].view(1, -1, 1, 1)) * math.sqrt(2),
                   _cl(br.get(('conv0', r))))
        w1 = p[k + 'conv1.weight'] / math.sqrt(9 * c)
        u1 = (F.conv2d(_depthwise(a, f, 1, True), w1, stride=2) + p[k + 'conv1.bias'].view(1, -1, 1, 1)) \
            * (math.sqrt(2) * (math.sqrt(2) / 2))
        x = y + _lrelu(u1, _cl(br.get(('conv1', r))))
    # 4x4 epilogue: minibatch std over groups of 4 (images j, j + B/4, ...), conv, fc, out, cmap
    B = x.shape[0]
    s = x.reshape(4, -1, 1, 512, 4, 4)
    s = (s - s.mean(dim=0)).square().mean(dim=0)
    s = (s + 1e-8).sqrt().mean(dim=[2, 3, 4]).reshape(-1, 1, 1, 1).repeat(4, 1, 4, 4)
    x = torch.cat([x, s], dim=1)
    wc = p['b4.conv.weight'] / math.sqrt(513 * 9)
    x = _lrelu((F.conv2d(x, wc, padding=1) + p['b4.conv.bias'].view(1, -1, 1, 1)) * math.sqrt(2),
               br.get('b4.conv'))
    x = _lrelu((F.linear(x.flatten(1), p['b4.fc.weight'] / math.sqrt(8192), p['b4.fc.bias'])) * math.sqrt(2),
               br.get('b4.fc'))
    x = F.linear(x, p['b4.out.weight'] / math.sqrt(512), p['b4.out.bias'])
    if cmap is not None:
        x = (x * cmap).sum(dim=1, keepdim=True) / math.sqrt(cmap.shape[1])
    return x


def make_params(R, nc, conditional, seed=0, dtype=torch.float32):
    """Backbone parameters by state_dict name with the module's init scales (randn weights) and
    small random biases (zero biases would leave the bias gradients' paths untested)."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    p = {}
    for i, r in enumerate(block_resolutions(R)):
        c, co = channels(r), channels(r // 2)
        k = 'b%d.' % r
        if i == 0:
            p[k + 'fromrgb.weight'], p[k + 'fromrgb.bias'] = rnd(c, nc, 1, 1), 0.1 * rnd(c)
        p[k + 'conv0.weight'], p[k + 'conv0.bias'] = rnd(c, c, 3, 3), 0.1 * rnd(c)
        p[k + 'conv1.weight'], p[k + 'conv1.bias'] = rnd(co, c, 3, 3), 0.1 * rnd(co)
        p[k + 'skip.weight'] = rnd(co, c, 1, 1)
    n = 512 if conditional else 1
    p['b4.conv.weight'], p['b4.conv.bias'] = rnd(512, 513, 3, 3), 0.1 * rnd(512)
    p['b4.fc.weight'], p['b4.fc.bias'] = rnd(512, 8192), 0.1 * rnd(512)
    p['b4.out.weight'], p['b4.out.bias'] = rnd(n, 512), 0.1 * rnd(n)
    return {k: v.to(dtype) for k, v in p.items()}


def names(R):
    """The parameter names in the kernels' order (nerf_from_image_b200.discriminator.parameters_of)."""
    rs = block_resolutions(R)
    out = ['b%d.fromrgb.weight' % R, 'b%d.fromrgb.bias' % R]
    for r in rs:
        out += ['b%d.%s' % (r, n) for n in ('conv0.weight', 'conv0.bias', 'conv1.weight', 'conv1.bias',
                                             'skip.weight')]
    return out + ['b4.conv.weight', 'b4.conv.bias', 'b4.fc.weight', 'b4.fc.bias', 'b4.out.weight', 'b4.out.bias']
