"""Tensor-core (wgmma) decoder tile (TriplanarDecoder.net) vs torch fp32 and vs the SIMT path."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from nerf_from_image_b200 import _lib

pytestmark = pytest.mark.gpu


def run_decoder(feats, w1, b1, w2, b2, A, mode):
    lib = _lib.load()
    nout = 1 + (A if A > 0 else 3)
    out = torch.full((feats.shape[0], nout), float('nan'), device='cuda')
    ws = torch.empty(32768, dtype=torch.uint8, device='cuda')
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.nfi_decoder_forward(p(feats), feats.shape[0], p(w1), p(b1), p(w2), p(b2), A,
                                       p(out), mode, p(ws), st))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('A', [10, 0, 15])
@pytest.mark.parametrize('n', [128, 1000, 128 * 4 * 150 + 77])
def test_decoder_tc_matches_fp32(cuda_lib, A, n):
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(n + A)
    nout = 1 + (A if A > 0 else 3)
    feats = (torch.randn(n, 32, generator=g) * 2).cuda()
    w1 = (torch.randn(64, 32, generator=g) / 32 ** 0.5).cuda()
    b1 = torch.randn(64, generator=g).cuda()
    w2 = (torch.randn(nout, 64, generator=g) / 8).cuda()
    b2 = torch.randn(nout, generator=g).cuda()
    ref = F.linear(F.softplus(F.linear(feats.double(), w1.double(), b1.double())),
                   w2.double(), b2.double())
    simt = run_decoder(feats, w1, b1, w2, b2, A, _lib.MLP_FP32_SIMT)
    tcv = run_decoder(feats, w1, b1, w2, b2, A, _lib.MLP_TC_3XTF32)
    assert torch.isfinite(tcv).all()
    e_simt = (simt.double() - ref).abs().max().item()
    e_tc = (tcv.double() - ref).abs().max().item()
    print('max abs err  simt %.2e  tc %.2e' % (e_simt, e_tc))
    assert e_simt < 2e-5
    assert e_tc < 2e-5     # single-pass TF32 would be ~3e-3 here
