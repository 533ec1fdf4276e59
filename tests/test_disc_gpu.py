"""The fused discriminator backbone (nfi_disc.cu) on the GPU against the float64 oracle
(oracle/disc_oracle.py):

1. logits and the gradients to the image, cmap and every parameter group, on the kernel's own
   leaky-ReLU branches, at B = 4, 8 and 32, nc 3 and 4, conditional and unconditional, 128^2 and
   64^2, and 256^2 (128 channels in the first block) (B = 32 at 128^2 has far more conv tiles than
   the GPU has SMs); beside them, the module's own fp32 arithmetic against plain float64;
2. determinism: two backward calls give the same bits, and a minibatch-std group of 4 images gives
   the same logits alone and inside a batch of 32;
3. through enable_fused_discriminator on the reference Discriminator (conditional pose, nc 4,
   B = 8, 64^2), against the module in float64 (its conditioning vector and mapping network, the
   backbone restated by the oracle on the kernel's branches): a generator-step-shaped loss, a
   discriminator-step-shaped loss, and an R1-shaped call that runs the module itself, also on an
   nn.DataParallel replica.

The bar is 1e-4, which two groups miss (README 4.10): the out layer's weight gradient and, through
the opt-in, the mapping network's gradients (which come through cmap's).  The out layer's weight
gradient is a sum over images of g_b fc(x_b) (and cmap's of g_b out(x_b)) in which the images'
terms cancel, so the fc output's relative error (~5e-5) grows in it (up to 1.4e-4 measured on an
H100); those groups are held to 2e-4 so that a regression beyond the measured miss still fails."""
import copy

import pytest
import torch
import torch.nn.functional as F

from nerf_from_image_b200 import discriminator as FD
from oracle import disc_oracle as DO
from tests import disc_cases as DC
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BAR = 1e-4
LOOSE = ('b4.out.weight', 'backbone.b4.out.weight', 'backbone.mapping.')


def _run(B, R, nc, cond, seed=1, g_seed=2):
    """Fused logits and gradients (with the branches the kernels took) and the float64 oracle's on
    those branches and on its own."""
    p = {k: v.to(DEV).requires_grad_() for k, v in DO.make_params(R, nc, cond, seed=seed).items()}
    img = DC.image(B, nc, R, seed + 10).to(DEV).requires_grad_()
    cm = DC.cmap(B, seed + 20).to(DEV).requires_grad_() if cond else None
    ps = [p[k] for k in DO.names(R)]
    out = FD._DiscFunction.apply(1, img, cm, *ps)
    br = {k: v.double() for k, v in FD.saved_preactivations(out).items()}
    g = torch.randn(B, 1, generator=torch.Generator().manual_seed(g_seed), dtype=torch.float64).to(DEV)
    out.backward(g.float())
    fused = {'logits': out.detach()} | {'img': img.grad, **({'cmap': cm.grad} if cond else {})} \
        | {k: p[k].grad for k in DO.names(R)}
    res = []
    for branches in (br, None):
        pd = {k: v.detach().double().requires_grad_() for k, v in p.items()}
        imd = img.detach().double().requires_grad_()
        cmd = cm.detach().double().requires_grad_() if cond else None
        o = DO.backbone(pd, imd, cmd, branches)
        o.backward(g)
        res.append({'logits': o.detach(), 'img': imd.grad, **({'cmap': cmd.grad} if cond else {})}
                   | {k: pd[k].grad for k in DO.names(R)})
    # the module's own arithmetic: the same restatement in fp32, TF32 off, on its own branches
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        pf = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
        imf = img.detach().clone().requires_grad_()
        cmf = cm.detach().clone().requires_grad_() if cond else None
        o = DO.backbone(pf, imf, cmf)
        o.backward(g.float())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    eager = {'logits': o.detach(), 'img': imf.grad, **({'cmap': cmf.grad} if cond else {})} \
        | {k: pf[k].grad for k in DO.names(R)}
    return fused, res[0], res[1], eager


def _errors(fused, want):
    return {k: Hh.rel_l2(fused[k].double(), want[k]) for k in want}


CASES = [(4, 128, 4, True), (8, 128, 3, False), (32, 128, 4, True), (4, 64, 3, True), (8, 64, 4, False),
         (32, 64, 3, False), (4, 256, 3, True)]


@pytest.mark.parametrize('B, R, nc, cond', CASES)
def test_outputs_and_gradients_against_float64(B, R, nc, cond):
    fused, on_branches, plain, eager = _run(B, R, nc, cond)
    err = _errors(fused, on_branches)
    err_plain = _errors(fused, plain)
    err_eager = _errors(eager, plain)
    print('B %d R %d nc %d cond %d: on the kernel branches max %.2e (%s); against plain float64: fused '
          'max %.2e, eager fp32 max %.2e' % (B, R, nc, cond, max(err.values()), max(err, key=err.get),
                                            max(err_plain.values()), max(err_eager.values())))
    bad = {k: v for k, v in err.items() if not v <= (2 * BAR if k.startswith(LOOSE) else BAR)}
    assert not bad, bad


def test_backward_is_bit_exact_and_groups_are_batch_independent():
    R, nc = 64, 4
    p = {k: v.to(DEV) for k, v in DO.make_params(R, nc, True, seed=3).items()}
    ps = [p[k].clone().requires_grad_() for k in DO.names(R)]
    img = DC.image(32, nc, R, 4).to(DEV)
    cm = DC.cmap(32, 5).to(DEV)
    grads = []
    for _ in range(2):
        x = img.clone().requires_grad_()
        c = cm.clone().requires_grad_()
        for t in ps:
            t.grad = None
        out = FD._DiscFunction.apply(1, x, c, *ps)
        out.backward(torch.ones_like(out))
        grads.append([x.grad, c.grad] + [t.grad for t in ps])
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    with torch.no_grad():
        full = FD._DiscFunction.apply(0, img, cm, *ps)
        idx = torch.tensor([3, 11, 19, 27], device=DEV)   # the group of image 3: j + k B/4
        alone = FD._DiscFunction.apply(0, img[idx].contiguous(), cm[idx].contiguous(), *ps)
    assert torch.equal(alone, full[idx])


@pytest.fixture(scope='module')
def reference():
    mods = DC.reference_modules()
    if mods is None:
        pytest.skip('the reference discriminator is not staged (oracle/stage_disc_reference.py)')
    return mods


def _pair(reference, nc=4, R=64, seed=6):
    discriminator, _ = reference
    D = DC.seed_module(discriminator.Discriminator(R, nc, DC.DATASET_CONFIG, conditional_pose=True), seed)
    Dd = copy.deepcopy(D).double()
    D = FD.enable_fused_discriminator(D.to(DEV))
    return D, Dd.to(DEV)


def _criterion(x, real):
    return F.softplus(-x if real else x).mean()


def _float64_call(Dd, fused_out, img, pose, focal):
    """Dd's conditioning vector and mapping network in float64, then the oracle backbone on the
    branches the fused call behind ``fused_out`` took."""
    br = {k: v.double() for k, v in FD.saved_preactivations(fused_out).items()}
    pose_utils = __import__(type(Dd).__module__, fromlist=['pose_utils']).pose_utils
    cond = pose_utils.matrix_to_conditioning_vector(pose.double(), focal.double(), DC.DATASET_CONFIG['camera_flipped'])
    cmap = Dd.backbone.mapping(None, cond)
    p = {k[len('backbone.'):]: v for k, v in Dd.named_parameters() if not k.startswith('backbone.mapping.')}
    return DO.backbone(p, img, cmap, br)


def test_generator_step_through_the_opt_in(reference):
    D, Dd = _pair(reference)
    D.requires_grad_(False)
    Dd.requires_grad_(False)
    B = 8
    pose, focal = (t.to(DEV) for t in DC.poses(B, 7))
    img = DC.image(B, 4, 64, 8).to(DEV).requires_grad_()
    out = D(img, 0, pose, None, focal)
    imd = img.detach().double().requires_grad_()
    _criterion(_float64_call(Dd, out, imd, pose, focal), True).backward()
    _criterion(out, True).backward()
    err = Hh.rel_l2(img.grad.double(), imd.grad)
    print('G step: image gradient %.2e' % err)
    assert err <= BAR


def test_discriminator_step_through_the_opt_in(reference):
    D, Dd = _pair(reference)
    B = 8
    pose, focal = (t.to(DEV) for t in DC.poses(B, 9))
    real, fake = DC.image(B, 4, 64, 10).to(DEV), DC.image(B, 4, 64, 11).to(DEV)
    o_real, o_fake = D(real, 1, pose, None, focal), D(fake, 1, pose, None, focal)
    (_criterion(_float64_call(Dd, o_real, real.double(), pose, focal), True)
     + _criterion(_float64_call(Dd, o_fake, fake.double(), pose, focal), False)).backward()
    (_criterion(o_real, True) + _criterion(o_fake, False)).backward()
    want = dict(Dd.named_parameters())
    err = {k: Hh.rel_l2(t.grad.double(), want[k].grad) for k, t in D.named_parameters()}
    print('D step: parameter gradients', {k: '%.2e' % v for k, v in err.items()})
    bad = {k: v for k, v in err.items() if not v <= (2 * BAR if k.startswith(LOOSE) else BAR)}
    assert not bad, bad


def test_r1_call_runs_the_module(reference):
    D, _ = _pair(reference)
    E = FD.enable_fused_discriminator(copy.deepcopy(D), enabled=False)
    B = 8
    pose, focal = (t.to(DEV) for t in DC.poses(B, 12))
    img = DC.image(B, 4, 64, 13).to(DEV)
    res = []
    for m in (D, E):
        x = img.clone().requires_grad_()
        m.zero_grad(set_to_none=True)
        out = m(x, 1, pose, None, focal)
        assert out.grad_fn is not None and 'DiscFunction' not in type(out.grad_fn).__name__
        g, = torch.autograd.grad(out.sum(), x, create_graph=True)
        pen = g.reshape(B, -1).square().sum(dim=1).mean()
        (_criterion(out, True) + 2.5 * pen).backward()
        res.append([pen.detach()] + [t.grad for t in m.parameters()])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_r1_call_on_a_data_parallel_replica_runs_the_module(reference):
    D, _ = _pair(reference)
    E = FD.enable_fused_discriminator(copy.deepcopy(D), enabled=False)
    rep = torch.nn.parallel.replicate(D, [0])[0]   # what nn.DataParallel runs, on one GPU
    assert len(list(rep.parameters())) == 0
    B = 8
    pose, focal = (t.to(DEV) for t in DC.poses(B, 14))
    img = DC.image(B, 4, 64, 15).to(DEV)
    res = []
    for m in (rep, E):
        x = img.clone().requires_grad_()
        out = m(x, 1, pose, None, focal)
        g, = torch.autograd.grad(out.sum(), x, create_graph=True)
        res.append((out.detach(), g.detach()))
    for a, b in zip(*res):
        assert torch.equal(a, b)
