"""The SegFormer-backbone oracle and the fused module's host side, without a GPU:

1. the oracle against the reference's Segformer (models/segformer.py) in float64, shallow (depths 1
   per stage, out_features 32, B = 2, 64^2), in eval mode and in train mode with the module's own
   drop-path masks -- live where the reference is installed, else against its recorded output
   under tests/golden/reference/;
2. the drop-path draw of the fused forward leaves the generator in the state the module's own
   train forward leaves it, with the same masks;
3. the oracle's float64 gradient against torch.autograd.gradcheck on slices of a few parameters
   (through four fixed projections of the features);
4. enable_fused_segformer keeps the module's parameters and state_dict keys, survives replication,
   switches back, refuses malformed modules and out-of-envelope images, and hands the kernels the
   parameters in named_parameters() order."""
import os

import pytest
import torch
from torch import nn

from nerf_from_image_b200 import _lib
from nerf_from_image_b200 import segformer as FS
from oracle import segformer_oracle as SO
from tests import helpers as Hh
from tests.segformer_standin import load, make_segformer, reference_available

SHALLOW = (1, 1, 1, 1)


def _image(b, h, seed):
    return torch.randn(b, 3, h, h, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _pre_cast(m, x, seed):
    """The module's output before its closing ``.float()`` (segformer.py:275): linear_pred's, as
    the last interpolate to the same size is the identity."""
    got = []
    h = m.linear_pred.register_forward_hook(lambda mod, i, o: got.append(o))
    torch.manual_seed(seed)
    with torch.no_grad():
        out = m(x)
    h.remove()
    assert torch.equal(got[0].float(), out)
    return got[0]


@pytest.mark.parametrize('train', [False, True])
def test_segformer_oracle_matches_the_reference(request, train):
    p = SO.make_params(SHALLOW, 32, seed=1)
    x = _image(2, 64, seed=2)

    def run_reference():
        m = load(make_segformer(32, SHALLOW).double(), p).train(train)
        out = _pre_cast(m, x, 3)
        torch.manual_seed(3)
        scales = FS.drop_scales(m, 2, 'cpu', torch.float64)
        return {'features': out, 'scales': scales if scales is not None else torch.empty(0)}

    if reference_available():
        ref = Hh.reference_output(request, run_reference)
    else:   # the recorded output of the same call
        name = request.node.name.replace('[', '.').replace(']', '')
        ref = torch.load(os.path.join(Hh.REFERENCE_GOLDEN, name + '.pt'), weights_only=True)
    scales = list(ref['scales'].double()) if train else None
    if train:   # block 1.0 has p = 0; every other block draws two masks
        assert ref['scales'].shape == (8, 2) and torch.equal(ref['scales'][:2], torch.ones(2, 2))
    with torch.no_grad():
        want = SO.forward(p, SHALLOW, x, scales)
    assert want.shape == (2, 32, 16, 16)
    assert torch.allclose(want, ref['features'], rtol=1e-12, atol=1e-12)


@pytest.mark.skipif(not reference_available(), reason='needs the installed reference module')
def test_drop_path_draws_match_the_module_forward():
    m = make_segformer(64, (2, 1, 3, 1)).double().train()
    x = _image(3, 32, seed=4)
    out = _pre_cast(m, x, 5)
    state = torch.get_rng_state()
    torch.manual_seed(5)
    scales = FS.drop_scales(m, 3, 'cpu', torch.float64)
    assert torch.equal(torch.get_rng_state(), state)
    assert scales.shape == (14, 3)
    with torch.no_grad():
        want = SO.forward(dict(m.named_parameters()), (2, 1, 3, 1), x, list(scales))
    assert torch.allclose(want, out, rtol=1e-12, atol=1e-12)


def test_oracle_float64_gradient_passes_gradcheck():
    p = SO.make_params(SHALLOW, 64, seed=6, stress=True)
    x = _image(1, 32, seed=7)
    names = ['patch_embed1.norm.bias', 'block1.0.attn.kv.bias', 'block2.0.mlp.dwconv.dwconv.weight',
             'block3.0.attn.sr.bias', 'block4.0.attn.q.weight', 'linear_fuse.bias']
    base = {n: p[n].clone() for n in names}
    scales = [torch.full((1,), 1.25, dtype=torch.float64)] * 8
    proj = torch.randn(4, 1, 64, 8, 8, generator=torch.Generator().manual_seed(8), dtype=torch.float64)

    def fn(delta):
        q = dict(p)
        for i, n in enumerate(names):
            q[n] = (base[n].flatten() + torch.nn.functional.pad(delta[2 * i:2 * i + 2],
                                                                (0, base[n].numel() - 2))).view_as(base[n])
        return (SO.forward(q, SHALLOW, x, scales)[None] * proj).flatten(1).sum(1)

    delta = torch.zeros(2 * len(names), dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(fn, (delta,), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_enable_keeps_parameters_and_state_dict():
    m = make_segformer(64, SHALLOW)
    names = [n for n, _ in m.named_parameters()]
    keys = list(m.state_dict().keys())
    base = type(m)
    assert FS.enable_fused_segformer(m) is m
    assert type(m) is not base and isinstance(m, base)
    assert [n for n, _ in m.named_parameters()] == names and list(m.state_dict().keys()) == keys
    FS.enable_fused_segformer(m)   # idempotent
    assert type(m).__mro__[1] is base
    rep = m._replicate_for_data_parallel()   # nn.DataParallel's replicas keep the class
    assert type(rep) is type(m)
    FS.enable_fused_segformer(m, enabled=False)
    assert type(m) is base


def test_parameter_order_is_named_parameters():
    depths = (2, 1, 3, 2)
    m = make_segformer(128, depths)
    assert FS.layout(m) == (depths, 128)
    got = FS.parameters_of(m, depths)
    want = list(m.parameters())
    assert len(got) == len(want) == 16 + 20 * 6 + 16 * 2 + 8 + 12
    assert all(a is b for a, b in zip(got, want))
    assert FS.param_names(depths) == [n for n, _ in m.named_parameters()] == SO.param_names(depths)


def test_b5_has_1064_parameter_tensors():
    assert len(FS.param_names(SO.B5_DEPTHS)) == 1064


def _refused(m, match):
    with pytest.raises(_lib.NfiError, match=match):
        FS.enable_fused_segformer(m)


def test_malformed_modules_are_refused():
    m = make_segformer(64, SHALLOW)
    m.block1[0].attn.q = nn.Linear(64, 32)
    _refused(m, 'block1.0')
    m = make_segformer(64, SHALLOW)
    m.block2[0].attn.sr_ratio = 2
    _refused(m, 'block2.0')
    m = make_segformer(64, SHALLOW)
    m.block3[0].norm1 = nn.GroupNorm(1, 320)
    _refused(m, 'block3.0')
    m = make_segformer(64, SHALLOW)
    m.norm4 = nn.LayerNorm(512)   # eps 1e-5 instead of the stage norm's 1e-6
    _refused(m, 'norm4')
    m = make_segformer(64, SHALLOW)
    m.patch_embed2.proj = nn.Conv2d(64, 96, 3, stride=2, padding=1)
    _refused(m, 'patch_embed2')
    _refused(make_segformer(32, SHALLOW), 'linear_pred')


def test_images_outside_the_envelope_are_refused():
    m = FS.enable_fused_segformer(make_segformer(64, SHALLOW))
    for shape in ((2, 3, 64, 96), (2, 3, 48, 48), (2, 3, 288, 288), (2, 1, 64, 64)):
        with pytest.raises(_lib.NfiError, match='images must be'):
            m(torch.zeros(shape))
    with pytest.raises(_lib.NfiError, match='image'):
        m(torch.zeros(2, 3, 64, 64, requires_grad=True))
    with pytest.raises(_lib.NfiError, match='CUDA'):
        m(torch.zeros(2, 3, 64, 64))
