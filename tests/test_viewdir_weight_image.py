"""The weight image of the view-conditioned pipelined forward kernel (csrc/nfi_layout.h), built on
the CPU by the very code the device runs (tests/c/vd_image_check.cpp) and un-permuted here from a
restatement of the layout: SWIZZLE_128B tiles, K positions in register-fragment order, W2's feature
rows at output columns 0..31 and the distance at 32, W3 at columns 1..A, TF32 hi + lo parts.
Evaluating the decoder from the un-permuted image reproduces
W3 . lrelu(vf + W2[1:] h + b2[1:]) + b3 and W2[0] h + b2[0] in float64."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'nerf_from_image_b200', 'csrc')

W1HI, W1LO, W2HI, W2LO, W3HI, W3LO = 0, 8192, 16384, 26624, 36864, 38912
B1, B2F, HEAD, BYTES = 40960, 41216, 41344, 41408
LOG2E = 1.4426950408889634


def sw128(row, chunk):
    return (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4)


def kpos(j):
    """Hidden unit j of a block of 8 sits where the accumulator fragment puts it when it is reused
    as an A fragment: units 2t, 2t + 1 at K positions t, t + 4."""
    t, odd = (j % 8) // 2, j % 2
    return (j // 8) * 8 + t + 4 * odd


@pytest.fixture(scope='module')
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('vd') / 'vd_image_check')
    subprocess.run(['g++', '-std=c++17', '-O1', '-Wall', '-Wextra', '-Werror', '-I', CSRC,
                    os.path.join(ROOT, 'tests', 'c', 'vd_image_check.cpp'), '-o', exe], check=True)
    return exe


def build_image(checker, tmp_path, A, scale1, scale3, pad, w):
    src, dst = str(tmp_path / 'w.bin'), str(tmp_path / 'img.bin')
    np.concatenate([np.array([A, scale1, scale3, pad], np.float32)] +
                   [x.astype(np.float32).ravel() for x in w]).tofile(src)
    subprocess.run([checker, src, dst], check=True)
    img = np.fromfile(dst, np.uint8)
    assert img.size == BYTES
    return img.view(np.float32)


def unpermute(img, A):
    f = lambda byte: float(img[byte // 4])
    nl = A if A > 0 else 3
    w1 = np.array([[f(W1HI + sw128(j, k >> 2) + (k & 3) * 4) + f(W1LO + sw128(j, k >> 2) + (k & 3) * 4)
                    for k in range(32)] for j in range(64)])
    def w2_at(col, j, base):
        jp = kpos(j)
        return f(base + (jp >> 5) * 5120 + sw128(col, (jp & 31) >> 2) + (jp & 3) * 4)
    w2 = np.array([[w2_at(col, j, W2HI) + w2_at(col, j, W2LO) for j in range(64)]
                   for col in range(40)])
    def w3_at(col, c, base):
        cp = kpos(c)
        return f(base + sw128(col, cp >> 2) + (cp & 3) * 4)
    w3 = np.array([[w3_at(col, c, W3HI) + w3_at(col, c, W3LO) for c in range(32)]
                   for col in range(16)])
    hi_parts = img[W1HI // 4:W1LO // 4].view(np.uint32)
    assert not (hi_parts & 0x1FFF).any(), 'hi parts must be exact in TF32'
    b1 = img[B1 // 4:B1 // 4 + 64].astype(np.float64)
    b2f = img[B2F // 4:B2F // 4 + 32].astype(np.float64)
    head = img[HEAD // 4:HEAD // 4 + 16].astype(np.float64)
    return w1, b1, w2, b2f, w3, head, nl


@pytest.mark.parametrize('A,scale3,pad', [(10, LOG2E, -1e30), (15, LOG2E, -1e30), (0, 1.0, 0.0)])
def test_unpermuted_image_reproduces_the_view_conditioned_decoder(checker, tmp_path, A, scale3, pad):
    rng = np.random.default_rng(4 + A)
    nl = A if A > 0 else 3
    w1, b1 = rng.standard_normal((64, 32)) / 6, 0.1 * rng.standard_normal(64)
    w2, b2 = rng.standard_normal((33, 64)) / 8, 0.1 * rng.standard_normal(33)
    w3, b3 = rng.standard_normal((nl, 32)) / 6, 0.1 * rng.standard_normal(nl)
    ws = [x.astype(np.float32).astype(np.float64) for x in (w1, b1, w2, b2, w3, b3)]
    w1, b1, w2, b2, w3, b3 = ws
    img = build_image(checker, tmp_path, A, LOG2E, scale3, pad, ws)
    i1, ib1, i2, ib2f, i3, head, _ = unpermute(img, A)

    x = rng.standard_normal((50, 32))
    vf = rng.standard_normal((50, 32))
    softplus = lambda v: np.logaddexp(v, 0.0)
    lrelu = lambda v: np.where(v > 0, v, 0.2 * v)
    h = softplus(x @ w1.T + b1)
    want_d = h @ w2[0] + b2[0]
    want_logits = lrelu(vf + h @ w2[1:].T + b2[1:]) @ w3.T + b3

    # as the kernel evaluates it: layer 1 in log2 units, D2 = [features | distance | zeros],
    # D3 column 0 = distance, columns 1.. = logits, + head
    h_img = np.log(2.0) * np.logaddexp2((x @ i1.T + ib1), 0.0)
    d2 = h_img @ i2.T
    assert np.all(d2[:, 33:] == 0)
    y = lrelu(d2[:, :32] + vf + ib2f)
    d3 = y @ i3.T
    assert np.all(d3[:, 0] == 0), 'column 0 of layer 3 carries no weights'
    got_d = d2[:, 32] + head[0]
    got_logits = (d3[:, 1:1 + nl] + head[1:1 + nl]) / scale3
    assert np.abs(got_d - want_d).max() < 1e-6
    assert np.abs(got_logits - want_logits).max() < 1e-6
    assert np.all(d3[:, 1 + nl:] == 0) and np.all(head[1 + nl:] == np.float32(pad))
