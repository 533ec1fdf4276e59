"""The synthesis parameter backward without a GPU: the per-layer restatement in the kernels'
decomposition (tests/synthesis_param_backward_oracle.py) against float64 autograd through
oracle.synthesis_oracle, and the C ABI of the parameter backward (struct mirror, exports, error
paths, workspace sizing)."""
import ctypes
import os
import re

import pytest
import torch

from oracle import synthesis_oracle as SO
from tests import synthesis_param_backward_oracle as SP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize('up', [False, True])
@pytest.mark.parametrize('with_noise', [False, True])
@pytest.mark.parametrize('cin,cout,h,batch', [(32, 64, 4, 2), (64, 32, 8, 3)])
def test_layer_decomposition_equals_autograd(up, with_noise, cin, cout, h, batch):
    g = torch.Generator().manual_seed(cin + cout + h + 7 * up + 3 * with_noise)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    pre, D = 'b8.conv0', 48
    p = {pre + '.weight': rn(cout, cin, 3, 3), pre + '.affine.weight': rn(cin, D),
         pre + '.affine.bias': 1 + 0.1 * rn(cin), pre + '.bias': 0.2 * rn(cout)}
    p = {k: v.requires_grad_() for k, v in p.items()}
    x = rn(batch, cin, h, h)
    w = rn(batch, D)
    H = 2 * h if up else h
    noise = (0.07 * rn(batch, 1, H, H)).requires_grad_() if with_noise else None
    dy = rn(batch, cout, H, H)
    y = SO.synthesis_layer(p, pre, x, w, noise, up, SO.fir_kernel(dtype=torch.float64))
    names = ['weight', 'bias', 'affine.weight', 'affine.bias']
    inputs = [p[pre + '.' + n] for n in names] + ([noise] if with_noise else [])
    want = torch.autograd.grad(y, inputs, dy)
    got = SP.layer_param_grads({k: v.detach() for k, v in p.items()}, pre, x, w,
                               noise.detach() if with_noise else None, up, dy)
    for n, t in zip(names + (['noise'] if with_noise else []), want):
        assert _rel(got[n], t) < 1e-10, (n, _rel(got[n], t))


def test_torgb_decomposition_equals_autograd():
    g = torch.Generator().manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    pre, D, cin, batch, h = 'b8.torgb', 48, 64, 2, 8
    p = {pre + '.weight': rn(96, cin, 1, 1), pre + '.affine.weight': rn(cin, D),
         pre + '.affine.bias': 1 + 0.1 * rn(cin), pre + '.bias': 0.2 * rn(96)}
    p = {k: v.requires_grad_() for k, v in p.items()}
    x, w, dimg = rn(batch, cin, h, h), rn(batch, D), rn(batch, 96, h, h)
    y = SO.to_rgb(p, pre, x, w)
    names = ['weight', 'bias', 'affine.weight', 'affine.bias']
    want = torch.autograd.grad(y, [p[pre + '.' + n] for n in names], dimg)
    got = SP.torgb_param_grads({k: v.detach() for k, v in p.items()}, pre, x, w, dimg)
    for n, t in zip(names, want):
        assert _rel(got[n], t) < 1e-10, (n, _rel(got[n], t))


def test_param_grads_struct_mirrors_the_header():
    from nerf_from_image_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'nfi_synth.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    for cname, cls in (('nfi_synth_layer_grads', _lib.SynthLayerGrads),
                       ('nfi_synth_param_grads', _lib.SynthParamGrads)):
        body = re.search(r'typedef struct %s \{(.*?)\} %s;' % (cname, cname), src, re.S).group(1)
        fields = [re.search(r'(\w+)\s*(?:\[\w+\])?$', d.strip()).group(1)
                  for d in body.split(';') if d.strip()]
        assert fields == [f[0] for f in cls._fields_], cname
    ptr = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.SynthLayerGrads) == 5 * ptr
    assert ctypes.sizeof(_lib.SynthParamGrads) == (3 * _lib.SYNTH_MAX_BLOCKS * 5 + 1) * ptr
    assert _lib.SynthParamGrads.g_const.offset == 3 * _lib.SYNTH_MAX_BLOCKS * 5 * ptr


def test_param_backward_entry_points_fail_cleanly_and_size_their_workspace():
    from nerf_from_image_b200 import _lib
    lib = _lib.load()
    assert lib.nfi_synthesis_param_workspace_bytes(None) == 0
    P = _lib.SynthParams()
    G, PG = _lib.SynthGrads(), _lib.SynthParamGrads()
    assert lib.nfi_synthesis_backward_params(None, None, None, None) != 0
    assert lib.nfi_synthesis_backward_params(ctypes.byref(P), ctypes.byref(G), None, None) != 0
    assert b'param_grads' in lib.nfi_last_error()
    P.batch = 1
    assert lib.nfi_synthesis_backward_params(ctypes.byref(P), ctypes.byref(G), ctypes.byref(PG),
                                             None) != 0
    assert len(lib.nfi_last_error()) > 0
    chans = (64, 64, 32)
    P.batch, P.img_resolution, P.img_channels, P.w_dim = 2, 16, 96, 64
    P.num_blocks, P.num_ws = 3, 6
    for i, c in enumerate(chans):
        P.channels[i] = c
    saved = lib.nfi_synthesis_saved_workspace_bytes(ctypes.byref(P))
    param = lib.nfi_synthesis_param_workspace_bytes(ctypes.byref(P))
    # the rebuilt layer input (a bf16 pair of the largest activation) comes on top
    assert saved > 0 and param >= saved + 2 * 16 * 16 * 64 * 4
