"""The backward weight image of the view-conditioned pipelined kernel (csrc/nfi_layout.h,
vd_bwd_weight_image_fill), built on the CPU by the very code the device runs
(tests/c/vd_bwd_image_check.cpp) and un-permuted here from a restatement of the layout: SWIZZLE_128B
tiles, K positions of the register-fragment operands (dF, dpre) in fragment order, TF32 hi + lo
parts, W3 with a zero distance column and no log2 e.  The three GEMMs of the kernel's bwd half,
evaluated from the un-permuted image, reproduce W3^T dlogits, W2^T [dDist; dF] and W1^T dpre / 3 in
float64."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'nerf_from_image_b200', 'csrc')
HEADER = os.path.join(ROOT, 'include', 'nfi_render.h')

W1HI, W1LO, W2HI, W2LO, W3HI, W3LO, W2D, BYTES = 0, 8192, 16384, 24576, 32768, 36864, 40960, 41216


def sw128(row, chunk):
    return (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4)


def kpos(j):
    """Unit j of a block of 8 sits where the accumulator fragment puts it when it is reused as an A
    fragment: units 2t, 2t + 1 at K positions t, t + 4."""
    t, odd = (j % 8) // 2, j % 2
    return (j // 8) * 8 + t + 4 * odd


@pytest.fixture(scope='module')
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('vdb') / 'vd_bwd_image_check')
    subprocess.run(['g++', '-std=c++17', '-O1', '-Wall', '-Wextra', '-Werror', '-I', CSRC,
                    os.path.join(ROOT, 'tests', 'c', 'vd_bwd_image_check.cpp'), '-o', exe], check=True)
    return exe


def build_image(checker, tmp_path, A, w):
    src, dst = str(tmp_path / 'w.bin'), str(tmp_path / 'img.bin')
    np.concatenate([np.array([A], np.float32)] + [x.astype(np.float32).ravel() for x in w]).tofile(src)
    subprocess.run([checker, src, dst], check=True)
    img = np.fromfile(dst, np.uint8)
    assert img.size == BYTES
    return img.view(np.float32)


def unpermute(img):
    f = lambda byte: float(img[byte // 4])
    both = lambda hi, lo, off: f(hi + off) + f(lo + off)
    # W1^T / 3: [channel c][hidden j], two 4 KB K-blocks of hidden units
    w1t = np.array([[both(W1HI, W1LO, (kpos(j) >> 5) * 4096 + sw128(c, (kpos(j) & 31) >> 2) +
                          (kpos(j) & 3) * 4) for j in range(64)] for c in range(32)])
    # W2f^T: [hidden j][feature c]
    w2t = np.array([[both(W2HI, W2LO, sw128(j, kpos(c) >> 2) + (kpos(c) & 3) * 4)
                     for c in range(32)] for j in range(64)])
    # W3^T: [feature c][output o], natural K order
    w3t = np.array([[both(W3HI, W3LO, sw128(c, o >> 2) + (o & 3) * 4) for o in range(32)]
                    for c in range(32)])
    for lo, hi in ((W1HI, W1LO), (W2HI, W2LO), (W3HI, W3LO)):
        assert not (img[lo // 4:hi // 4].view(np.uint32) & 0x1FFF).any(), 'hi parts must be exact in TF32'
    w2d = img[W2D // 4:W2D // 4 + 64].astype(np.float64)
    return w1t, w2t, w3t, w2d


@pytest.mark.parametrize('A', [10, 15, 0])
def test_unpermuted_backward_image_reproduces_the_decoder_transposes(checker, tmp_path, A):
    rng = np.random.default_rng(40 + A)
    nl = A if A > 0 else 3
    w1 = rng.standard_normal((64, 32)) / 6
    w2 = rng.standard_normal((33, 64)) / 8
    w3 = rng.standard_normal((nl, 32)) / 6
    w1, w2, w3 = (x.astype(np.float32).astype(np.float64) for x in (w1, w2, w3))
    w1t, w2t, w3t, w2d = unpermute(build_image(checker, tmp_path, A, (w1, w2, w3)))

    n = 50
    dlogits = rng.standard_normal((n, nl))
    ddist = rng.standard_normal(n)
    # a D2 / dOut row as the shading warpgroup writes it: [dDist, dlogits, 0 ...]
    dout = np.zeros((n, 16))
    dout[:, 0], dout[:, 1:1 + nl] = ddist, dlogits
    assert np.all(w3t[:, 0] == 0), 'the distance column of W3 must carry no weight'
    assert np.all(w3t[:, 1 + nl:] == 0)
    dg = dout @ w3t[:, :16].T
    assert np.abs(dg - dlogits @ w3).max() < 1e-9   # unscaled W3: dlogits are natural units

    slope = np.where(rng.random((n, 32)) < 0.5, 1.0, 0.2)
    df = dg * slope
    d3 = df @ w2t.T + ddist[:, None] * w2d[None, :]
    assert np.abs(d3 - np.concatenate([ddist[:, None], df], axis=1) @ w2).max() < 1e-9

    dpre = rng.standard_normal((n, 64))
    w1_3 = (w1.astype(np.float32) * np.float32(1.0 / 3.0)).astype(np.float64)  # fp32 W1 / 3
    assert np.abs(dpre @ w1t.T - dpre @ w1_3).max() < 1e-9
    assert np.abs(dpre @ w1t.T - dpre @ w1 / 3).max() < 1e-6


def test_view_backward_workspace_constant_matches_the_header():
    """fused.py sizes a view-conditioned inversion backward's workspace (the forward and backward
    weight images, 48 KiB slots) with _lib.VIEW_BACKWARD_WORKSPACE_BYTES."""
    from nerf_from_image_b200 import _lib
    m = re.search(r'#define NFI_VIEW_BACKWARD_WORKSPACE_BYTES (\d+)', open(HEADER).read())
    assert m, 'NFI_VIEW_BACKWARD_WORKSPACE_BYTES missing from the header'
    assert int(m.group(1)) == _lib.VIEW_BACKWARD_WORKSPACE_BYTES
    layout = open(os.path.join(CSRC, 'nfi_layout.h')).read()
    off = int(re.search(r'constexpr int kVdBwdImageOffset = (\d+);', layout).group(1))
    assert 2 * off == _lib.VIEW_BACKWARD_WORKSPACE_BYTES and BYTES <= off
