"""The path-length regulariser's double backward without a GPU: the restatement in the kernels'
decomposition (tests/synthesis_hvp_oracle.py) against torch's float64 double backward through
oracle.synthesis_oracle, and the C ABI of nfi_synthesis_backward_hvp (struct mirror, exports,
error paths, scratch sizing)."""
import ctypes
import os
import re

import pytest
import torch

from oracle import synthesis_oracle as SO
from tests import synthesis_hvp_oracle as SH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ['weight', 'bias', 'affine.weight', 'affine.bias']


def _close(got, want, what):
    if want is None or want.norm().item() == 0.0:   # Phi does not depend on it
        assert got.abs().max().item() == 0.0, what
        return
    err = ((got - want).norm() / want.norm()).item()
    assert err < 1e-10, (what, err)


def _rn(g):
    return lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)


@pytest.mark.parametrize('up', [False, True])
@pytest.mark.parametrize('with_noise', [False, True])
@pytest.mark.parametrize('cin,cout,h,batch', [(32, 64, 4, 2), (64, 32, 8, 3)])
def test_layer_hvp_equals_double_backward(up, with_noise, cin, cout, h, batch):
    rn = _rn(torch.Generator().manual_seed(cin + cout + h + 7 * up + 3 * with_noise))
    pre, D = 'b8.conv0', 48
    p = {pre + '.weight': rn(cout, cin, 3, 3), pre + '.affine.weight': rn(cin, D),
         pre + '.affine.bias': 1 + 0.1 * rn(cin), pre + '.bias': 0.2 * rn(cout)}
    p = {k: v.requires_grad_() for k, v in p.items()}
    x, w, t = rn(batch, cin, h, h), rn(batch, D).requires_grad_(), rn(batch, D)
    H = 2 * h if up else h
    noise = (0.07 * rn(batch, 1, H, H)).requires_grad_() if with_noise else None
    dy = rn(batch, cout, H, H)
    f = SO.fir_kernel(dtype=torch.float64)
    y = SO.synthesis_layer(p, pre, x, w, noise, up, f)
    (gw,) = torch.autograd.grad((y * dy).sum(), w, create_graph=True)
    inputs = [p[pre + '.' + n] for n in NAMES] + [w] + ([noise] if with_noise else [])
    want = torch.autograd.grad((gw * t).sum(), inputs, allow_unused=True)
    pd = {k: v.detach() for k, v in p.items()}
    L, _, _ = SH.layer_forward(pd, pre, x, None, w.detach(), t,
                               noise.detach() if with_noise else None, up, f)
    _, _, got = SH.layer_backward(L, dy, torch.zeros_like(dy), f)
    for n, wt in zip(NAMES + ['ws'] + (['noise'] if with_noise else []), want):
        _close(got[n], wt, n)


def test_torgb_hvp_equals_double_backward():
    rn = _rn(torch.Generator().manual_seed(5))
    pre, D, cin, batch, h = 'b8.torgb', 48, 64, 2, 8
    p = {pre + '.weight': rn(96, cin, 1, 1), pre + '.affine.weight': rn(cin, D),
         pre + '.affine.bias': 1 + 0.1 * rn(cin), pre + '.bias': 0.2 * rn(96)}
    p = {k: v.requires_grad_() for k, v in p.items()}
    x, w, t, dimg = rn(batch, cin, h, h), rn(batch, D).requires_grad_(), rn(batch, D), rn(batch, 96, h, h)
    (gw,) = torch.autograd.grad((SO.to_rgb(p, pre, x, w) * dimg).sum(), w, create_graph=True)
    want = torch.autograd.grad((gw * t).sum(), [p[pre + '.' + n] for n in NAMES] + [w],
                               allow_unused=True)
    _, _, _, got = SH.torgb_hvp({k: v.detach() for k, v in p.items()}, pre, x, torch.zeros_like(x),
                                w.detach(), t, dimg)
    for n, wt in zip(NAMES + ['ws'], want):
        _close(got[n], wt, n)


def _net(channels, D, seed, noise_layers=()):
    """A small random network in extract_params' layout; resolutions 4 .. 4 * 2^(n-1)."""
    rn = _rn(torch.Generator().manual_seed(seed))
    res = [4 << i for i in range(len(channels))]
    p, layers = {}, {}

    def layer(pre, cin, cout, k):
        p[pre + '.weight'] = rn(cout, cin, k, k)
        p[pre + '.affine.weight'] = rn(cin, D)
        p[pre + '.affine.bias'] = 1 + 0.1 * rn(cin)
        p[pre + '.bias'] = 0.2 * rn(cout)

    for i, (r, c) in enumerate(zip(res, channels)):
        pre = 'b%d' % r
        if i == 0:
            p[pre + '.const'] = rn(c, 4, 4)
        else:
            layer(pre + '.conv0', channels[i - 1], c, 3)
            layers[pre + '.conv0'] = dict(use_noise=pre + '.conv0' in noise_layers, up=True)
        layer(pre + '.conv1', c, c, 3)
        layers[pre + '.conv1'] = dict(use_noise=pre + '.conv1' in noise_layers, up=False)
        layer(pre + '.torgb', c, 96, 1)
    p['meta'] = dict(img_resolution=res[-1], img_channels=96, w_dim=D, resolutions=res, layers=layers)
    return p, rn


@pytest.mark.parametrize('channels,noise_layers', [
    ((64,), ('b4.conv1',)),                                       # the b4.const block alone
    ((64, 32, 32), ('b4.conv1', 'b8.conv0', 'b16.conv1')),        # a whole small network
])
def test_network_hvp_equals_double_backward(channels, noise_layers):
    D, B = 40, 2
    p, rn = _net(channels, D, 11 + len(channels), noise_layers)
    R, num_ws = p['meta']['img_resolution'], 2 * len(channels) + 1   # one row nothing reads
    ws, t = rn(B, num_ws, D).requires_grad_(), rn(B, num_ws, D)
    res = lambda k: int(k.split('.')[0][1:])
    noises = {k: (0.1 * rn(B, 1, res(k), res(k))).requires_grad_() for k in noise_layers}
    n = rn(B, 96, R, R)
    names = [k for k in p if k != 'meta']
    pg = {k: p[k].clone().requires_grad_() for k in names}
    pg['meta'] = p['meta']
    img = SO.synthesis_forward(pg, ws, noises)
    (gws,) = torch.autograd.grad((img * n).sum(), ws, create_graph=True)
    inputs = [ws] + [pg[k] for k in names] + list(noises.values())
    want = torch.autograd.grad((gws * t).sum(), inputs, allow_unused=True)
    g_ws, grads, g_noise = SH.synthesis_hvp(p, ws.detach(), {k: v.detach() for k, v in noises.items()},
                                            n, t)
    _close(g_ws, want[0], 'ws')
    assert g_ws[:, -1].abs().max().item() == 0.0   # the row the network does not read
    for k, wt in zip(names, want[1:1 + len(names)]):
        _close(grads[k], wt, k)
    for k, wt in zip(noises, want[1 + len(names):]):
        _close(g_noise[k], wt, k)


def test_hvp_struct_mirrors_the_header():
    from nerf_from_image_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'nfi_synth.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    body = re.search(r'typedef struct nfi_synth_hvp \{(.*?)\} nfi_synth_hvp;', src, re.S).group(1)
    fields = [re.search(r'(\w+)$', d.strip()).group(1) for d in body.split(';') if d.strip()]
    assert fields == [f[0] for f in _lib.SynthHvp._fields_]
    ptr = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.SynthHvp) == 4 * ptr + ctypes.sizeof(ctypes.c_size_t)
    for name in ('nfi_synthesis_hvp_scratch_bytes', 'nfi_synthesis_backward_hvp'):
        assert re.search(r'NFI_API\s+\w+\s+%s\(' % name, src), name
        assert name in _lib.EXPORTS


def test_hvp_entry_points_fail_cleanly_and_size_their_scratch():
    from nerf_from_image_b200 import _lib
    lib = _lib.load()
    assert lib.nfi_synthesis_hvp_scratch_bytes(None) == 0
    P, H, PG = _lib.SynthParams(), _lib.SynthHvp(), _lib.SynthParamGrads()
    assert lib.nfi_synthesis_backward_hvp(None, None, None, None) != 0
    assert lib.nfi_synthesis_backward_hvp(ctypes.byref(P), None, None, None) != 0
    assert b'hvp' in lib.nfi_last_error()
    P.batch = 1
    assert lib.nfi_synthesis_backward_hvp(ctypes.byref(P), ctypes.byref(H), ctypes.byref(PG),
                                          None) != 0
    assert len(lib.nfi_last_error()) > 0
    chans = (64, 64, 32)
    P.img_resolution, P.img_channels, P.w_dim = 16, 96, 64
    P.num_blocks, P.num_ws = 3, 6
    for i, c in enumerate(chans):
        P.channels[i] = c
    sizes = []
    for b in (1, 2, 4):
        P.batch = b
        sizes.append(lib.nfi_synthesis_hvp_scratch_bytes(ctypes.byref(P)))
    assert 0 < sizes[0] < sizes[1] < sizes[2]
