"""The synthesis backward without a GPU: the restatement in the kernels' decomposition
(tests/synthesis_backward_oracle.py) against autograd through oracle.synthesis_oracle in float64,
and the C ABI of the backward (struct mirror, exports, error paths)."""
import ctypes
import os
import re

import pytest
import torch

from fixtures import synthetic
from oracle import synthesis_oracle as SO
from tests import helpers_synth as HS
from tests import synthesis_backward_oracle as SB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _double(p):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v)
            for k, v in p.items()}


def _autograd(p, ws, noises, g_img):
    ws = ws.clone().requires_grad_()
    img = SO.synthesis_forward(p, ws, noises)
    return torch.autograd.grad(img, ws, g_img)[0]


@pytest.mark.parametrize('channels,batch', [((32, 32, 32), 2), ((64, 32, 64, 32), 1)])
def test_decomposition_equals_autograd(channels, batch):
    res = 4 << (len(channels) - 1)
    p = _double(synthetic.make_synthesis_params(11, res, channels, 64))
    g = torch.Generator().manual_seed(12)
    ws = torch.randn(batch, 2 * len(channels), 64, generator=g, dtype=torch.float64)
    g_img = torch.randn(batch, 96, res, res, generator=g, dtype=torch.float64)
    noises = {k: v.double() for k, v in HS.const_noises(p).items()}
    assert noises, 'the seeded net has noise on every layer'
    want = _autograd(p, ws, noises, g_img)
    got = SB.synthesis_backward(p, ws, noises, g_img)
    err = ((got - want).norm() / want.norm()).item()
    assert err < 1e-10, err
    # every row is reached (shared rows: ToRGB of block i and conv0 of block i+1)
    assert (want.norm(dim=-1) > 0).all()


def test_decomposition_on_a_fixture_without_noise():
    p, ws, _, _ = HS.load_case('synth_mixed_nonoise')
    p = _double(p)
    ws = ws.double()
    R = p['meta']['img_resolution']
    g_img = torch.randn(ws.shape[0], 96, R, R, generator=torch.Generator().manual_seed(2),
                        dtype=torch.float64)
    want = _autograd(p, ws, {}, g_img)
    got = SB.synthesis_backward(p, ws, {}, g_img)
    assert ((got - want).norm() / want.norm()).item() < 1e-10


def test_grads_struct_mirrors_the_header():
    from nerf_from_image_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'nfi_synth.h')).read()
    body = re.search(r'typedef struct nfi_synth_grads \{(.*?)\} nfi_synth_grads;', src, re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = [re.search(r'(\w+)\s*$', d.strip()).group(1) for d in body.split(';') if d.strip()]
    assert fields == [f[0] for f in _lib.SynthGrads._fields_] == ['g_planes', 'g_ws']
    assert ctypes.sizeof(_lib.SynthGrads) == 2 * ctypes.sizeof(ctypes.c_void_p)


def test_backward_entry_points_are_exported_and_fail_cleanly():
    from nerf_from_image_b200 import _lib
    lib = _lib.load()
    for name in ('nfi_synthesis_saved_workspace_bytes', 'nfi_synthesis_forward_saved',
                 'nfi_synthesis_backward'):
        assert name in _lib.EXPORTS and hasattr(lib, name), name
    assert lib.nfi_synthesis_saved_workspace_bytes(None) == 0
    P = _lib.SynthParams()   # all zero: inconsistent resolution
    assert lib.nfi_synthesis_saved_workspace_bytes(ctypes.byref(P)) == 0
    assert lib.nfi_synthesis_forward_saved(None, None) != 0
    assert lib.nfi_synthesis_forward_saved(ctypes.byref(P), None) != 0
    assert len(lib.nfi_last_error()) > 0
    G = _lib.SynthGrads()
    assert lib.nfi_synthesis_backward(ctypes.byref(P), None, None) != 0
    assert b'grads' in lib.nfi_last_error()
    P.batch = 1
    assert lib.nfi_synthesis_backward(ctypes.byref(P), ctypes.byref(G), None) != 0
    assert len(lib.nfi_last_error()) > 0


def test_saved_workspace_covers_the_plain_one():
    """Sizing only (no device memory is touched): the saved forward's workspace holds the plain
    forward's plus the pre-activations (at least one fp32 value per layer output)."""
    from nerf_from_image_b200 import _lib
    lib = _lib.load()
    P = _lib.SynthParams()
    chans = (64, 64, 32)
    P.batch, P.img_resolution, P.img_channels, P.w_dim = 2, 16, 96, 64
    P.num_blocks, P.num_ws = 3, 6
    for i, c in enumerate(chans):
        P.channels[i] = c
    plain = lib.nfi_synthesis_workspace_bytes(ctypes.byref(P))
    saved = lib.nfi_synthesis_saved_workspace_bytes(ctypes.byref(P))
    u = sum(2 * (4 << i) ** 2 * c * 4 * (2 if i else 1) for i, c in enumerate(chans))
    assert plain > 0 and saved >= plain + u
