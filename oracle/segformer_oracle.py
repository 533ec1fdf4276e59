"""Functional float64 restatement of the bootstrap encoder's SegFormer backbone (the reference's
models/segformer.py:175-275, ``Segformer.forward``) -- TEST / BASELINE INFRASTRUCTURE.

``forward(p, depths, img, scales)`` takes the parameters as a dict keyed by the module's own
``named_parameters()`` names and the drop-path scales explicitly: ``scales[2k]`` and
``scales[2k + 1]`` are the [B] factors of block k's attention and MLP branches (blocks counted
across the stages), or None for 1.  Written in its own words from the layer definitions; the
decoder head is computed as the module computes it (upsample, concatenate, then linear_fuse).
"""
import math

import torch
import torch.nn.functional as F

DIMS = (64, 128, 320, 512)
HEADS = (1, 2, 5, 8)
SR = (8, 4, 2, 1)
DECODER = 768
B5_DEPTHS = (3, 6, 40, 3)


def param_names(depths):
    """The module's named_parameters() names, in order."""
    names = []
    for i in range(4):
        names += ['patch_embed%d.%s' % (i + 1, n) for n in ('proj.weight', 'proj.bias', 'norm.weight', 'norm.bias')]
    for i in range(4):
        for k in range(depths[i]):
            b = 'block%d.%d.' % (i + 1, k)
            ns = ['norm1', 'attn.q', 'attn.kv', 'attn.proj'] + (['attn.sr', 'attn.norm'] if SR[i] > 1 else []) + [
                'norm2', 'mlp.fc1', 'mlp.dwconv.dwconv', 'mlp.fc2']
            for n in ns:
                names += [b + n + '.weight', b + n + '.bias']
        names += ['norm%d.weight' % (i + 1), 'norm%d.bias' % (i + 1)]
    for i in reversed(range(4)):
        names += ['linear_c%d.proj.weight' % (i + 1), 'linear_c%d.proj.bias' % (i + 1)]
    names += ['linear_fuse.weight', 'linear_fuse.bias', 'linear_pred.weight', 'linear_pred.bias']
    return names


def _ln(x, p, name, eps):
    return F.layer_norm(x, x.shape[-1:], p[name + '.weight'], p[name + '.bias'], eps)


def _branch(y, s):
    return y if s is None else y * s.to(y).view(-1, 1, 1)


def _attention(p, b, x, r, sr, heads):
    B, N, C = x.shape
    d = C // heads
    q = F.linear(x, p[b + 'q.weight'], p[b + 'q.bias']).view(B, N, heads, d).transpose(1, 2)
    src = x
    if sr > 1:
        m = x.transpose(1, 2).reshape(B, C, r, r)
        m = F.conv2d(m, p[b + 'sr.weight'], p[b + 'sr.bias'], stride=sr)
        src = _ln(m.flatten(2).transpose(1, 2), p, b + 'norm', 1e-5)
    kv = F.linear(src, p[b + 'kv.weight'], p[b + 'kv.bias']).view(B, -1, 2, heads, d).permute(2, 0, 3, 1, 4)
    logits = torch.matmul(q, kv[0].transpose(-2, -1)) / math.sqrt(d)
    o = torch.matmul(torch.softmax(logits, dim=-1), kv[1]).transpose(1, 2).reshape(B, N, C)
    return F.linear(o, p[b + 'proj.weight'], p[b + 'proj.bias'])


def _mlp(p, b, x, r):
    B, N, _ = x.shape
    h = F.linear(x, p[b + 'fc1.weight'], p[b + 'fc1.bias'])
    C4 = h.shape[-1]
    h = F.conv2d(h.transpose(1, 2).reshape(B, C4, r, r), p[b + 'dwconv.dwconv.weight'],
                 p[b + 'dwconv.dwconv.bias'], padding=1, groups=C4)
    h = F.gelu(h.flatten(2).transpose(1, 2))
    return F.linear(h, p[b + 'fc2.weight'], p[b + 'fc2.bias'])


def forward(p, depths, img, scales=None):
    """features [B,out,H/4,W/4] of the backbone with parameters ``p`` on ``img`` [B,3,H,W]."""
    B = img.shape[0]
    x = img
    feats = []
    k = 0
    for i in range(4):
        pe = 'patch_embed%d.' % (i + 1)
        st, pad = (4, 3) if i == 0 else (2, 1)
        x = F.conv2d(x, p[pe + 'proj.weight'], p[pe + 'proj.bias'], stride=st, padding=pad)
        r = x.shape[-1]
        t = _ln(x.flatten(2).transpose(1, 2), p, pe + 'norm', 1e-5)
        for j in range(depths[i]):
            b = 'block%d.%d.' % (i + 1, j)
            sa = scales[2 * k] if scales is not None else None
            sm = scales[2 * k + 1] if scales is not None else None
            t = t + _branch(_attention(p, b + 'attn.', _ln(t, p, b + 'norm1', 1e-6), r, SR[i], HEADS[i]), sa)
            t = t + _branch(_mlp(p, b + 'mlp.', _ln(t, p, b + 'norm2', 1e-6), r), sm)
            k += 1
        t = _ln(t, p, 'norm%d' % (i + 1), 1e-6)
        x = t.reshape(B, r, r, -1).permute(0, 3, 1, 2)
        feats.append(x)
    r0 = feats[0].shape[-1]
    cat = []
    for i in reversed(range(4)):
        f = feats[i]
        c = F.linear(f.flatten(2).transpose(1, 2), p['linear_c%d.proj.weight' % (i + 1)],
                     p['linear_c%d.proj.bias' % (i + 1)])
        c = c.transpose(1, 2).reshape(B, -1, f.shape[2], f.shape[3])
        if i > 0:
            c = F.interpolate(c, size=(r0, r0), mode='bilinear', align_corners=False)
        cat.append(c)
    x = F.conv2d(torch.cat(cat, dim=1), p['linear_fuse.weight'], p['linear_fuse.bias'])
    return F.conv2d(x, p['linear_pred.weight'], p['linear_pred.bias'])


def make_params(depths, out_features, seed, dtype=torch.float64, init='reference', stress=False):
    """Seeded parameters keyed by name.  ``init='reference'`` follows ``Segformer._init_weights``
    (normal convs with fan-out std, truncated-normal 0.02 linears, zero biases, unit LayerNorms);
    ``'default'`` draws PyTorch's default layer init scale (uniform, 1/sqrt(fan_in)) for every
    weight and bias.  ``stress`` perturbs it towards trained statistics: LayerNorm weights
    ~ N(1, 0.5^2), biases ~ N(0, 0.2^2), and weights at 3x scale."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    shapes = shapes_of(depths, out_features)
    for n in param_names(depths):
        shape = shapes[n]
        is_ln = n.endswith('.weight') and len(shape) == 1
        if n.endswith('.bias'):
            fan_in = _fan_in(shapes[n[:-5] + '.weight'])
            if stress:
                t = torch.randn(shape, generator=g, dtype=torch.float64) * 0.2
            elif init == 'default' and not _is_ln(n, shapes):
                t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(fan_in)
            else:
                t = torch.zeros(shape, dtype=torch.float64)
        elif is_ln:
            t = 1 + torch.randn(shape, generator=g, dtype=torch.float64) * 0.5 if stress else torch.ones(shape, dtype=torch.float64)
        else:
            if init == 'default':
                t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(_fan_in(shape))
            elif len(shape) == 4:
                fan_out = shape[0] * shape[2] * shape[3] // (shape[0] if shape[1] == 1 else 1)
                t = torch.randn(shape, generator=g, dtype=torch.float64) * math.sqrt(2.0 / fan_out)
            else:
                t = torch.fmod(torch.randn(shape, generator=g, dtype=torch.float64), 2.0) * 0.02
            if stress:
                t = t * 3
        p[n] = t.to(dtype)
    return p


def _fan_in(shape):
    return int(torch.tensor(shape[1:]).prod().item()) if len(shape) > 1 else 1


def _is_ln(n, shapes):
    return len(shapes[n[:-5] + '.weight']) == 1


def shapes_of(depths, out_features):
    """Each parameter's shape, keyed by name."""
    s = {}
    for i in range(4):
        C, Cp = DIMS[i], (3 if i == 0 else DIMS[i - 1])
        k = 7 if i == 0 else 3
        pe = 'patch_embed%d.' % (i + 1)
        s[pe + 'proj.weight'], s[pe + 'proj.bias'] = (C, Cp, k, k), (C,)
        s[pe + 'norm.weight'], s[pe + 'norm.bias'] = (C,), (C,)
        for j in range(depths[i]):
            b = 'block%d.%d.' % (i + 1, j)
            lin = {'attn.q': (C, C), 'attn.kv': (2 * C, C), 'attn.proj': (C, C), 'mlp.fc1': (4 * C, C),
                   'mlp.fc2': (C, 4 * C)}
            for n, sh in lin.items():
                s[b + n + '.weight'], s[b + n + '.bias'] = sh, (sh[0],)
            for n in ('norm1', 'norm2') + (('attn.norm',) if SR[i] > 1 else ()):
                s[b + n + '.weight'], s[b + n + '.bias'] = (C,), (C,)
            if SR[i] > 1:
                s[b + 'attn.sr.weight'], s[b + 'attn.sr.bias'] = (C, C, SR[i], SR[i]), (C,)
            s[b + 'mlp.dwconv.dwconv.weight'], s[b + 'mlp.dwconv.dwconv.bias'] = (4 * C, 1, 3, 3), (4 * C,)
        s['norm%d.weight' % (i + 1)], s['norm%d.bias' % (i + 1)] = (C,), (C,)
        s['linear_c%d.proj.weight' % (i + 1)], s['linear_c%d.proj.bias' % (i + 1)] = (DECODER, C), (DECODER,)
    s['linear_fuse.weight'], s['linear_fuse.bias'] = (DECODER, 4 * DECODER, 1, 1), (DECODER,)
    s['linear_pred.weight'], s['linear_pred.bias'] = (out_features, DECODER, 1, 1), (out_features,)
    return s
