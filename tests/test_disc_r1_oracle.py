"""The R1 double backward's float64 decomposition (tests/disc_r1_oracle.py), without a GPU:

1. against torch's float64 double backward through oracle/disc_oracle.py to 1e-10: the minibatch
   std alone, the 4x4 epilogue alone, one block (with a loss whose g-dot of the block output is not
   zero), and a whole backbone at 16^2, nc 3 and 4, conditional and unconditional; the epilogue
   biases' R1 gradients are exactly zero;
2. the oracle's R1 penalty and gradients against the unmodified reference ``Discriminator`` (the
   penalty step of run.py), live where the reference is staged, else against its recorded output
   under tests/golden/reference/;
3. the R1 opt-in's bookkeeping: routing with and without ``r1``, and the flag on a simulated
   ``nn.DataParallel`` replica."""
import copy
import os

import pytest
import torch

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.discriminator import enable_fused_discriminator
from oracle import disc_oracle as DO
from tests import disc_cases as DC
from tests import disc_r1_oracle as RO
from tests import helpers as Hh
from tests.test_disc_oracle import _module, _replica

TOL = 1e-10
F64 = torch.float64


def _rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=F64)


def _rel(a, b):
    n = b.norm()
    return ((a - b).norm() / n).item() if n > 0 else a.norm().item()


def test_minibatch_std_alone():
    B = 8
    x = _rnd(1, B, 512, 4, 4)
    dx, gxs = _rnd(2, B, 512, 4, 4), _rnd(3, B, 513, 4, 4)
    xr = x.clone().requires_grad_()
    sd, xs = RO.mbstd(xr)
    g, = torch.autograd.grad((xs * gxs).sum(), xr, create_graph=True)
    assert _rel(RO.mbstd_backward(gxs, x), g.detach()) < TOL
    h, = torch.autograd.grad((g * dx).sum(), xr)
    assert _rel(RO.mbstd_hvp(gxs, x, dx), h) < TOL
    dsd_want = torch.func.jvp(lambda v: RO.mbstd(v)[0], (x,), (dx,))[1]
    assert _rel(RO.mbstd_tangent(x, dx)[0], dsd_want) < TOL
    # and the std restated as disc_oracle's backbone takes it
    s = x.reshape(4, -1, 1, 512, 4, 4)
    s = (s - s.mean(dim=0)).square().mean(dim=0)
    assert _rel(sd, (s + 1e-8).sqrt().mean(dim=[2, 3, 4]).reshape(-1)) < TOL


@pytest.mark.parametrize('cond', [False, True])
def test_epilogue_alone(cond):
    B = 8
    p = DO.make_params(8, 4, cond, seed=4, dtype=F64)
    x4, dx4 = _rnd(5, B, 512, 4, 4), _rnd(6, B, 512, 4, 4)
    cm = _rnd(7, B, 512) if cond else None
    gl = _rnd(8, B, 1)
    got, g, dg, _ = RO.epilogue_r1(p, x4, cm, gl, dx4)
    names = [k for k in p if k.startswith('b4.')]
    pd = {k: p[k].clone().requires_grad_() for k in names}
    xr = x4.clone().requires_grad_()
    cr = cm.clone().requires_grad_() if cond else None
    glr = gl.clone().requires_grad_()
    lg = RO.epilogue_forward(pd, xr, cr)['logits']
    g_want, = torch.autograd.grad((lg * glr).sum(), xr, create_graph=True)
    assert _rel(g, g_want.detach()) < TOL
    (g_want * dx4).sum().backward()
    assert _rel(dg, xr.grad) < TOL
    for k in names:
        want = pd[k].grad if pd[k].grad is not None else torch.zeros_like(p[k])
        assert _rel(got[k], want) < TOL, k
    assert _rel(got['g_logits'], glr.grad) < TOL
    if cond:
        assert _rel(got['cmap'], cr.grad) < TOL
    for k in ('b4.conv.bias', 'b4.fc.bias', 'b4.out.bias'):
        assert torch.count_nonzero(got[k]) == 0


def test_one_block():
    """Block b16 of a 16^2 backbone under L = <G, y> + c/2 |y|^2, so that g_y = G + c y and
    g-dot_y = c y-dot are both non-zero."""
    B, c = 4, 0.5
    p = DO.make_params(16, 3, False, seed=9, dtype=F64)
    k = 'b16.'
    x = _rnd(10, B, 512, 16, 16)
    t = _rnd(11, B, 512, 16, 16)
    G = _rnd(12, B, 512, 8, 8)
    names = [n for n in p if n.startswith(k) and 'fromrgb' not in n]
    pd = {n: p[n].clone().requires_grad_() for n in names}
    xr = x.clone().requires_grad_()
    y = RO.block_forward(pd, k, xr)['y']
    gx, = torch.autograd.grad((G * y).sum() + 0.5 * c * y.square().sum(), xr, create_graph=True)
    (gx * t).sum().backward()
    s = RO.block_forward(p, k, x)
    tg = RO.block_tangent(s, t)
    got, g_x, dg_x = RO.block_r1(s, tg, k, G + c * s['y'], c * tg['dy'])
    assert _rel(g_x, gx.detach()) < TOL
    assert _rel(dg_x, xr.grad) < TOL
    for n in names:
        assert _rel(got[n], pd[n].grad) < TOL, n


@pytest.mark.parametrize('cond', [False, True])
@pytest.mark.parametrize('nc', [3, 4])
def test_whole_backbone(nc, cond):
    B, R = 4, 16
    p = DO.make_params(R, nc, cond, seed=13, dtype=F64)
    img, t = DC.image(B, nc, R, 14, dtype=F64), DC.image(B, nc, R, 15, dtype=F64)
    cm = DC.cmap(B, 16, dtype=F64) if cond else None
    gl = _rnd(17, B, 1)
    got = RO.r1(p, img, cm, gl, t)
    want = RO.double_backward(p, img, cm, gl, t)
    err = {k: _rel(got[k], want[k]) for k in want}
    assert max(err.values()) < TOL, err
    for k in ('b4.conv.bias', 'b4.fc.bias', 'b4.out.bias'):
        assert torch.count_nonzero(got[k]) == 0


def _summary(grads):
    """Each gradient as its norm and four projections on fixed random directions (what the recorded
    output keeps: the full tensors of a 16^2 backbone are hundreds of MB in float64)."""
    out = {}
    for i, (k, g) in enumerate(sorted(grads.items())):
        v = _rnd(100 + i, 4, g.numel())
        out[k] = torch.cat([g.reshape(1, -1).norm(dim=1), v @ g.reshape(-1)])
    return out


def test_oracle_matches_the_reference_r1_penalty(request):
    """run.py's penalty step (d_grad_real with create_graph, penalty = mean |d_grad_real_b|^2,
    (r1/2 penalty).backward()) on the reference Discriminator in float64 (conditional pose, nc 4,
    B = 4, 16^2, the backbone's parameters from oracle/disc_oracle.make_params), against the
    oracle's decomposition on the same cmap."""
    B, R, r1 = 4, 16, 10.0
    pose, focal = (t.double() for t in DC.poses(B, 18))
    img = DC.image(B, 4, R, 19, dtype=F64)
    p = DO.make_params(R, 4, True, seed=22, dtype=F64)

    def run_reference():
        D = _module().double()
        DC.load_backbone(D.backbone, p)
        x = img.clone().requires_grad_()
        out = D(x, 1, pose, None, focal)
        g, = torch.autograd.grad(out.sum(), x, create_graph=True)
        pen = g.reshape(B, -1).square().sum(dim=1).mean()
        (r1 / 2 * pen).backward()
        bb = D.backbone
        pose_utils = __import__(type(D).__module__, fromlist=['pose_utils']).pose_utils
        with torch.no_grad():
            cmap = bb.mapping(None, pose_utils.matrix_to_conditioning_vector(
                pose, focal, DC.DATASET_CONFIG['camera_flipped']))
        # (the epilogue biases are not on the penalty's graph: no .grad, an exact zero)
        grads = {k[len('backbone.'):]: v.grad if v.grad is not None else torch.zeros_like(v)
                 for k, v in D.named_parameters() if not k.startswith('backbone.mapping.')}
        return {'penalty': pen.detach(), 'cmap': cmap, 'img': x.grad, 'grads': _summary(grads)}

    if DC.reference_staged():
        ref = Hh.reference_output(request, run_reference)
    else:
        name = request.node.name.replace('[', '.').replace(']', '')
        ref = torch.load(os.path.join(Hh.REFERENCE_GOLDEN, name + '.pt'), weights_only=True)
    cm = ref['cmap']
    x = img.clone().requires_grad_()
    g, = torch.autograd.grad(DO.backbone(p, x, cm).sum(), x)
    pen = g.reshape(B, -1).square().sum(dim=1).mean()
    assert _rel(pen, ref['penalty']) < 1e-12
    got = RO.r1(p, img, cm, torch.ones(B, 1, dtype=F64), r1 * g / B)
    assert _rel(got['img'], ref['img']) < TOL
    mine = _summary({k: got[k] for k in p})
    assert sorted(mine) == sorted(ref['grads'])
    for k in p:
        assert _rel(mine[k], ref['grads'][k]) < TOL, k


def test_r1_opt_in_routing_and_the_flag_on_a_replica():
    D = _module()
    pose, focal = DC.poses(4, 20)
    img = DC.image(4, 4, 16, 21)
    E = enable_fused_discriminator(copy.deepcopy(D))
    assert not getattr(E, '_nfi_r1', False)
    x = img.clone().requires_grad_()
    assert torch.equal(E(x, 1, pose, None, focal), D(x, 1, pose, None, focal))   # the module
    F_ = enable_fused_discriminator(copy.deepcopy(D), r1=True)
    assert F_._nfi_r1 and type(F_) is type(E)
    with pytest.raises(_lib.NfiError, match='CUDA'):     # the R1 call now takes the fused path
        F_(img.clone().requires_grad_(), 1, pose, None, focal)
    rep = _replica(F_)
    assert len(list(rep.parameters())) == 0 and rep._nfi_r1
    with pytest.raises(_lib.NfiError, match='CUDA'):
        rep(img.clone().requires_grad_(), 1, pose, None, focal)
    rep0 = _replica(E)
    x, y = img.clone().requires_grad_(), img.clone().requires_grad_()
    assert torch.equal(rep0(x, 1, pose, None, focal), D(y, 1, pose, None, focal))
    # switching back, or re-enabling without r1, drops the flag
    assert not hasattr(enable_fused_discriminator(F_, r1=False), '_nfi_r1')
    G = enable_fused_discriminator(copy.deepcopy(D), r1=True)
    assert not hasattr(enable_fused_discriminator(G, enabled=False), '_nfi_r1')
