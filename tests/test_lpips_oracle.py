"""The LPIPS-VGG oracle and the fused module's host side, without a GPU:

1. the oracle's taps against torchvision's vgg16().features on the same random weights;
2. the oracle's float64 gradient against torch.autograd.gradcheck on a 16^2 image;
3. the oracle against the reference-layout stand-in module (tests/lpips_standin.py);
4. FusedLPIPS reads its weights from that layout, carries them as buffers, and refuses what it
   does not serve (CPU tensors, the one-tensor and cached-feature forms)."""
import pytest
import torch

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.lpips import FusedLPIPS, extract_weights
from oracle import lpips_oracle as LO
from tests.lpips_standin import StandInLPIPSLoss


def _images(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, h, w, generator=g) * 2 - 1


def test_oracle_taps_match_torchvision_vgg16():
    tv = pytest.importorskip('torchvision')
    p = LO.make_weights(seed=1)
    feats = tv.models.vgg16(weights=None).features.eval()
    convs = [m for m in feats if isinstance(m, torch.nn.Conv2d)]
    with torch.no_grad():
        for m, w, b in zip(convs, p['conv_w'], p['conv_b']):
            m.weight.copy_(w)
            m.bias.copy_(b)
        x = _images(2, 32, 48, seed=2)
        h = (x - p['shift'].view(1, 3, 1, 1)) / p['scale'].view(1, 3, 1, 1)
        want, cuts = [], (0, 4, 9, 16, 23, 30)
        for k in range(5):
            h = feats[cuts[k]:cuts[k + 1]](h)
            want.append(h.clone())
        got = LO.features(p, x)
    for a, b in zip(got, want):
        assert a.shape == b.shape
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-5), (a - b).abs().max()


def test_oracle_matches_the_reference_layout_stand_in():
    p = LO.make_weights(seed=3)
    m = StandInLPIPSLoss(p)
    x, y = _images(3, 32, 32, seed=4), _images(3, 32, 32, seed=5)
    with torch.no_grad():
        want = m(x, y)
        got = LO.distance(p, x, y)
        mean = m(x, y, reduction='mean')
    assert want.shape == (3, 1)
    assert torch.allclose(got, want[:, 0], rtol=1e-5, atol=1e-7)
    assert torch.allclose(mean, want.mean())


def test_oracle_float64_gradient_passes_gradcheck():
    p = LO.make_weights(seed=6, dtype=torch.float64)
    x = _images(1, 16, 16, seed=7).double().requires_grad_()
    y = _images(1, 16, 16, seed=8).double()
    assert torch.autograd.gradcheck(lambda a: LO.distance(p, a, y), (x,), eps=1e-6, atol=1e-7,
                                    rtol=1e-4)


def test_oracle_branch_overrides_reproduce_the_plain_forward():
    p = LO.make_weights(seed=9, dtype=torch.float64)
    x, y = _images(2, 32, 32, seed=10).double(), _images(2, 32, 32, seed=11).double()
    _, u0 = LO.features(p, x, with_u=True)
    _, u1 = LO.features(p, y, with_u=True)
    a = LO.distance(p, x, y)
    b = LO.distance(p, x, y, LO.branches_from_u(u0), LO.branches_from_u(u1))
    assert torch.equal(a, b)


def test_zero_feature_vectors_have_a_zero_gradient_in_the_oracle():
    p = LO.make_weights(seed=12, dtype=torch.float64)
    p['conv_b'][12] = p['conv_b'][12] - 1e3     # relu5_3 is zero everywhere
    x = _images(1, 32, 32, seed=13).double().requires_grad_()
    y = _images(1, 32, 32, seed=14).double()
    d = LO.distance(p, x, y)
    d.sum().backward()
    assert torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0
    taps0 = LO.features(p, x.detach())
    assert taps0[4].abs().max() == 0


def test_weights_are_extracted_from_the_reference_layout():
    p = LO.make_weights(seed=15)
    m = StandInLPIPSLoss(p)
    shift, scale, cw, cb, lw = extract_weights(m)
    assert torch.equal(shift, p['shift']) and torch.equal(scale, p['scale'])
    assert all(torch.equal(a, b) for a, b in zip(cw, p['conv_w']))
    assert all(torch.equal(a, b) for a, b in zip(cb, p['conv_b']))
    assert all(torch.equal(a, b) for a, b in zip(lw, p['lin']))
    f = FusedLPIPS(m)
    names = dict(f.named_buffers())
    assert len(names) == 2 + 2 * 13 + 5
    assert torch.equal(names['conv12_weight'], p['conv_w'][12])
    assert torch.equal(names['lin4_weight'], p['lin'][4])
    assert f.to(torch.float64).shift.dtype == torch.float64   # buffers follow .to()


def test_fused_module_refusals_without_a_gpu():
    f = FusedLPIPS(StandInLPIPSLoss(LO.make_weights(seed=16)))
    x = _images(1, 16, 16, seed=17)
    with pytest.raises(_lib.NfiError):
        f(x, x)                       # CPU tensors: there is no CPU path
    with pytest.raises(_lib.NfiError):
        f(x)                          # features only
    with pytest.raises(_lib.NfiError):
        f(x, (x,))                    # cached features
    bad =StandInLPIPSLoss(LO.make_weights(seed=16))
    bad.lpips.net.slice5 = torch.nn.Sequential()
    with pytest.raises(_lib.NfiError):
        FusedLPIPS(bad)
