"""The encoder-heads oracle and the fused module's host side, without a GPU:

1. the oracle against the reference's BootstrapEncoder (models/encoder.py, random init,
   pretrained=False, the backbone replaced by given features) in float64 -- live where the
   reference is installed, else against its recorded output under tests/golden/reference/;
2. the oracle's float64 gradient against torch.autograd.gradcheck on a narrow instance;
3. enable_fused_encoder keeps the module's parameters and state_dict keys, survives replication,
   switches back, and refuses malformed heads and CPU tensors."""
import os

import pytest
import torch
from torch import nn

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.encoder import enable_fused_encoder
from oracle import encoder_oracle as EO
from tests import helpers as Hh
from tests.encoder_standin import (FixedFeatures, StandInBootstrapEncoder, load_params,
                                   reference_encoder, seed_linear)

LATENT = 64


def _reference_staged():
    from oracle import reference_lift as RL
    from oracle import stage_encoder_reference
    return RL.available() and stage_encoder_reference.available(RL.REFERENCE_ROOT)


def _features(b, h, w, seed, c=512):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, c, h, w, generator=g, dtype=torch.float64)


@pytest.mark.parametrize('separate', [False, True])
def test_oracle_matches_the_reference_module(request, separate):
    p = EO.make_params(seed=1, dtype=torch.float64)
    f = _features(2, 4, 6, seed=2)
    fl = _features(2, 4, 6, seed=3) if separate else f

    def run_reference():
        enc = reference_encoder(LATENT, separate_backbones=separate)
        enc.backbone = FixedFeatures(f)
        if separate:
            enc.backbone_latent = FixedFeatures(fl)
        load_params(enc.double(), p, post_seed=4)
        with torch.no_grad():
            coords, seg, w = enc(torch.zeros(2, 3, 16, 24, dtype=torch.float64))
        return {'coords': coords, 'segmentation': seg, 'w': w}

    if _reference_staged():
        ref = Hh.reference_output(request, run_reference)
    else:   # the recorded output of the same call
        name = request.node.name.replace('[', '.').replace(']', '')
        ref = torch.load(os.path.join(Hh.REFERENCE_GOLDEN, name + '.pt'), weights_only=True)
    maps, pooled = EO.heads(p, f, fl)
    post = seed_linear(StandInBootstrapEncoder(LATENT).w_regressor_post.double(), 4)
    with torch.no_grad():
        w = post(pooled).unsqueeze(1)
    assert torch.allclose(maps[:, :3].permute(0, 2, 3, 1), ref['coords'], rtol=1e-12, atol=1e-12)
    assert torch.allclose(torch.sigmoid(maps[:, 3]), ref['segmentation'], rtol=1e-12, atol=1e-12)
    assert torch.allclose(w, ref['w'], rtol=1e-12, atol=1e-12)


def test_oracle_float64_gradient_passes_gradcheck():
    p = EO.make_params(seed=5, channels=4, dtype=torch.float64)
    f = _features(1, 2, 3, seed=6, c=4).requires_grad_()
    fl = _features(1, 2, 3, seed=7, c=4).requires_grad_()
    ws = [p[k].clone().requires_grad_() for k in EO.NAMES]

    def fn(f, fl, *ws):
        maps, pooled = EO.heads(dict(zip(EO.NAMES, ws)), f, fl)
        return maps, pooled

    assert torch.autograd.gradcheck(fn, (f, fl, *ws), eps=1e-6, atol=1e-7, rtol=1e-4)


def test_branch_overrides_reproduce_the_plain_forward():
    p = EO.make_params(seed=8, channels=8, dtype=torch.float64)
    f, fl = _features(2, 3, 5, seed=9, c=8), _features(2, 3, 5, seed=10, c=8)
    u = EO.pre_activations(p, f, fl)
    br = {k: v > 0 for k, v in u.items()}
    a, b = EO.heads(p, f, fl), EO.heads(p, f, fl, br)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('kw', [{}, {'latent_regressor': False}, {'pose_regressor': False},
                                {'separate_backbones': True}])
def test_enable_keeps_parameters_and_state_dict(kw):
    enc = StandInBootstrapEncoder(LATENT, **kw)
    params = list(enc.parameters())
    keys = list(enc.state_dict().keys())
    enable_fused_encoder(enc)
    assert type(enc).__name__ == 'FusedStandInBootstrapEncoder'
    assert isinstance(enc, StandInBootstrapEncoder)
    assert all(a is b for a, b in zip(enc.parameters(), params)) and len(list(enc.parameters())) == len(params)
    assert list(enc.state_dict().keys()) == keys
    # nn.DataParallel's replicas are copies of the instance's class
    rep = enc._replicate_for_data_parallel()
    assert type(rep) is type(enc)
    enable_fused_encoder(enc, False)
    assert type(enc) is StandInBootstrapEncoder
    enable_fused_encoder(enable_fused_encoder(enc))   # idempotent
    assert type(enc).__name__ == 'FusedStandInBootstrapEncoder'


def test_malformed_heads_are_refused():
    enc = StandInBootstrapEncoder(LATENT)
    enc.post[2] = nn.Conv2d(512, 512, 3, padding=2)
    with pytest.raises(_lib.NfiError):
        enable_fused_encoder(enc)
    enc = StandInBootstrapEncoder(LATENT)
    enc.post[1] = nn.LeakyReLU(0.2)
    with pytest.raises(_lib.NfiError):
        enable_fused_encoder(enc)
    enc = StandInBootstrapEncoder(LATENT)
    enc.w_regressor_pre = nn.Sequential(nn.Conv2d(512, 256, 3, padding=1), nn.ReLU())
    with pytest.raises(_lib.NfiError):
        enable_fused_encoder(enc)
    enc = StandInBootstrapEncoder(LATENT)
    enc.post[4] = nn.Conv2d(512, 4, 3, padding=1, bias=False)
    with pytest.raises(_lib.NfiError):
        enable_fused_encoder(enc)
    assert type(enc) is StandInBootstrapEncoder


def test_cpu_tensors_are_refused():
    enc = enable_fused_encoder(StandInBootstrapEncoder(LATENT))
    with pytest.raises(_lib.NfiError):
        enc(torch.zeros(1, 3, 16, 16))
