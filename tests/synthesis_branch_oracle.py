"""The synthesis network in float64 on chosen leaky-ReLU branches -- TEST INFRASTRUCTURE.

``synthesis_forward(p, ws, noises, masks)`` is ``oracle.synthesis_oracle.synthesis_forward`` with
each layer's activation written ``x = where(mask, u, 0.2 u)``: autograd, its double backward and
the parameter gradients then take the slope the mask chose at every position.  With masks
``u > 0`` of the same forward it is that forward, bit for bit, gradients included.

Why: a pre-activation u within rounding of zero has no reliable sign.  A forward that computes u
to ~1e-5 (bf16-pair operands, fp32 accumulation) may take the other branch than float64 at such a
position, and then its backward is the exact backward of a network that differs from the float64
one there; one such position can move ws.grad by 1e-3.  ``borrow_branches`` takes the kernel's
branch only where a bound on the kernel's forward error (asserted on every layer) says float64
cannot tell the sign either; everywhere else the truth is the plain float64 network.  (Signs that
differ put |u64| under |u_kernel - u64|, so the first bound implies the second; both are asserted.)

Layers are in the order the kernels run them: b4.conv1, b8.conv0, b8.conv1, ...; every ``u`` is
channel-first [B, C, res, res], as the reference's.
"""
import math

import torch

from oracle import synthesis_oracle as SO

# Bound on the kernel's forward error in u (absolute, asserted per layer at TAU / 4) and the |u64|
# under which a branch is borrowed.  Measured on an H100 (700 W): max |u_kernel - u64| per layer
# 2e-5 .. 2.0e-4 on the test nets (up to 13 blocks' worth of 32..256 channels, growing with the
# depth and K = 9 Cin), 6.5e-5 .. 3.7e-4 on the 512-channel 256^2 network; borrowed positions had
# |u64| <= 2.8e-5 and <= 8e-5.
TAU = 1e-3
TAU_FULL = 2e-3


def layer_names(p):
    names = []
    for r in p['meta']['resolutions']:
        names += ['b%d.conv1' % r] if r == 4 else ['b%d.conv0' % r, 'b%d.conv1' % r]
    return names


def synthesis_forward(p, ws, noises=None, masks=None):
    """-> (img [B, img_channels, R, R], [u of every layer]).  ``masks``: one boolean tensor per
    layer, shaped like its u (True: slope 1, False: slope 0.2), or None for the branches of this
    forward's own u."""
    meta = p['meta']
    f = SO.fir_kernel(ws.device, ws.dtype)
    noises = noises or {}
    x = img = None
    w_idx, us = 0, []

    def layer(key, x, w, up):
        s = SO.affine(p, key, w)
        u = SO.modulated_conv(x, p[key + '.weight'], s, noises.get(key), up, f)
        u = (u + p[key + '.bias'].view(1, -1, 1, 1)) * math.sqrt(2)
        mask = u > 0 if masks is None else masks[len(us)]
        us.append(u)
        return torch.where(mask, u, 0.2 * u)

    for r in meta['resolutions']:
        pre = 'b%d' % r
        if r == 4:
            x = p[pre + '.const'].unsqueeze(0).repeat(ws.shape[0], 1, 1, 1)
            n_conv = 1
        else:
            x = layer(pre + '.conv0', x, ws[:, w_idx], True)
            n_conv = 2
        x = layer(pre + '.conv1', x, ws[:, w_idx + n_conv - 1], False)
        y = SO.to_rgb(p, pre + '.torgb', x, ws[:, w_idx + n_conv])
        img = y if img is None else SO.upsample_img(img, f) + y
        w_idx += n_conv
    return img, us


def preactivations(p, ws, noises=None):
    """Every layer's u of the plain forward, without a graph."""
    with torch.no_grad():
        return synthesis_forward(p, ws, noises)[1]


def borrow_branches(p, u_kernel, u64, tau):
    """Masks of the kernel's branches, guarded: per layer max |u_kernel - u64| < tau / 4 (the
    kernel's forward error), and every position where the signs disagree has |u64| < tau, where
    float64 cannot vouch for its sign against that error.  ``u_kernel``: channel-last
    [B, res, res, C] (as ``nerf_from_image_b200.synthesis.saved_preactivations`` returns them),
    ``u64`` channel-first.  -> (masks, {layer: borrowed positions}); prints both per layer."""
    masks, borrowed, lines, checks = [], {}, [], []
    for name, uk, ud in zip(layer_names(p), u_kernel, u64):
        uk = uk.permute(0, 3, 1, 2).to(ud.device, torch.float64)
        assert uk.shape == ud.shape, (name, uk.shape, ud.shape)
        err = (uk - ud).abs().max().item()
        flip = (uk > 0) != (ud > 0)
        n = int(flip.sum())
        worst = ud[flip].abs().max().item() if n else 0.0
        lines.append('%s max|du| %.1e borrowed %d (max |u64| %.1e)' % (name, err, n, worst))
        checks.append((name, err, worst))
        masks.append(uk > 0)
        borrowed[name] = n
    print('  u vs float64 (tau %.0e): %s' % (tau, '; '.join(lines)))
    for name, err, worst in checks:
        assert err < tau / 4, (name, 'forward u error', err, 'bound', tau / 4)
        assert worst < tau, (name, 'a branch differs where |u64| =', worst)
    return masks, borrowed


def ws_grad(p, ws, noises, g_img, masks=None):
    """dL/dws of L = <g_img, img> in float64, on the masks' branches (plain with None)."""
    w = ws.detach().clone().requires_grad_()
    img = synthesis_forward(p, w, noises, masks)[0]
    return torch.autograd.grad(img, w, g_img)[0]


def max_rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def row_errors(got, want):
    """rel-L2 of every ws row (rows the network barely reads are taken relative to 1e-3 of the
    whole gradient)."""
    return ((got - want).norm(dim=(0, 2))
            / want.norm(dim=(0, 2)).clamp_min(1e-3 * want.norm())).tolist()


def kernel_branches(p, u_kernel, ws, noises=None, tau=None):
    """Float64 parameters / latents / noise from ``p`` (fp32), the plain forward's u, and the
    guarded masks of the kernel's branches -> (pd, wd, nz, masks, borrowed)."""
    pd = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in p.items()}
    wd = ws.double()
    nz = {k: v.double() for k, v in (noises or {}).items()}
    masks, borrowed = borrow_branches(p, u_kernel, preactivations(pd, wd, nz), tau or TAU)
    return pd, wd, nz, masks, borrowed
