"""The discriminator oracle and the fused module's host side, without a GPU:

1. the oracle against the reference's DiscriminatorBackbone (models/stylegan.py, unmodified) in
   float64, for nc 3 and 4, conditional and unconditional, 64^2 and 128^2 -- live where the
   reference is installed, else against its recorded output under tests/golden/reference/;
2. enable_fused_discriminator keeps the module's parameters and state_dict keys, switches back, and
   refuses CPU tensors; an R1-shaped call runs the module's forward."""
import copy
import os

import pytest
import torch

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.discriminator import enable_fused_discriminator
from oracle import disc_oracle as DO
from tests import disc_cases as DC
from tests import helpers as Hh


@pytest.mark.parametrize('R', [64, 128])
@pytest.mark.parametrize('cond', [False, True])
@pytest.mark.parametrize('nc', [3, 4])
def test_disc_oracle_matches_the_reference_backbone(request, nc, cond, R):
    B = 4
    p = DO.make_params(R, nc, cond, seed=1, dtype=torch.float64)
    img = DC.image(B, nc, R, 2, dtype=torch.float64)
    c = torch.randn(B, 13, generator=torch.Generator().manual_seed(3), dtype=torch.float64)

    def run_reference():
        _, stylegan = DC.reference_modules()
        bb = stylegan.DiscriminatorBackbone(13 if cond else 0, R, nc,
                                            mapping_kwargs={'lr_multiplier': 0.01, 'num_layers': 2,
                                                            'normalize_c': False}).double()
        DC.load_backbone(DC.seed_module(bb, 4), p)
        with torch.no_grad():
            cmap = bb.mapping(None, c) if cond else None
            return {'logits': bb(img, c if cond else None), 'cmap': cmap}

    if DC.reference_staged():
        ref = Hh.reference_output(request, run_reference)
    else:   # the recorded output of the same call
        name = request.node.name.replace('[', '.').replace(']', '')
        ref = torch.load(os.path.join(Hh.REFERENCE_GOLDEN, name + '.pt'), weights_only=True)
    got = DO.backbone(p, img, ref['cmap'])
    assert got.shape == (B, 1)
    assert Hh.rel_l2(got, ref['logits']) < 1e-12


def _module():
    mods = DC.reference_modules()
    if mods is None:
        pytest.skip('the reference discriminator is not staged (oracle/stage_disc_reference.py)')
    return DC.seed_module(mods[0].Discriminator(16, 4, DC.DATASET_CONFIG, conditional_pose=True), 5)


def test_opt_in_keeps_the_module_and_refuses_cpu_tensors():
    D = _module()
    keys = list(D.state_dict())
    params = list(D.parameters())
    E = enable_fused_discriminator(copy.deepcopy(D))
    assert type(E).__name__ == 'FusedDiscriminator' and isinstance(E, type(D))
    assert list(E.state_dict()) == keys
    assert [tuple(t.shape) for t in E.parameters()] == [tuple(t.shape) for t in params]
    pose, focal = DC.poses(4, 6)
    img = DC.image(4, 4, 16, 7)
    with pytest.raises(_lib.NfiError, match='CUDA'):
        E(img, 0, pose, None, focal)
    # R1-shaped (image and parameters require grad): the module's forward, here on the CPU
    x = img.clone().requires_grad_()
    assert torch.equal(E(x, 0, pose, None, focal), D(x, 0, pose, None, focal))
    assert type(enable_fused_discriminator(E, enabled=False)) is type(D)


def _replica(module):
    """A CPU stand-in for what ``torch.nn.parallel.replicate`` makes of ``module``: every submodule
    through ``_replicate_for_data_parallel`` (no registered parameters), the weights attached as
    plain tensors computed from the originals (as the broadcast copies are)."""
    mods = list(module.modules())
    copies = [m._replicate_for_data_parallel() for m in mods]
    index = {id(m): i for i, m in enumerate(mods)}
    for m, c in zip(mods, copies):
        for k, child in m._modules.items():
            c._modules[k] = copies[index[id(child)]] if child is not None else None
        for k, t in m._parameters.items():
            setattr(c, k, t * 1 if t is not None else None)
    return copies[0]


def test_r1_shaped_call_on_a_data_parallel_replica_runs_the_module():
    D = _module()
    E = enable_fused_discriminator(copy.deepcopy(D))
    rep = _replica(E)
    assert len(list(rep.parameters())) == 0 and type(rep) is type(E)
    pose, focal = DC.poses(4, 8)
    img = DC.image(4, 4, 16, 9)
    x, y = img.clone().requires_grad_(), img.clone().requires_grad_()
    got = rep(x, 1, pose, None, focal)      # on the CPU: the fused path would raise NfiError
    want = D(y, 1, pose, None, focal)
    assert torch.equal(got, want)
    gx, = torch.autograd.grad(got.sum(), x, create_graph=True)
    gy, = torch.autograd.grad(want.sum(), y, create_graph=True)
    assert torch.equal(gx, gy)
    # and with the replica's weights frozen (the generator step's shape) it takes the fused path
    with torch.no_grad():
        frozen = _replica(E)
    with pytest.raises(_lib.NfiError, match='CUDA'):
        frozen(img.clone().requires_grad_(), 0, pose, None, focal)
