"""The sm_90a SDF point evaluator (csrc/nfi_heads.cu through nfi_sdf_points_forward / _backward)
and the regulariser heads built on it (nerf_from_image_b200/heads.py) against the oracle
(oracle/heads_oracle.py, pinned to the reference Generator's own heads): values, first-order
gradients, and the gradients of the eikonal term -- a double backward in the reference, one
analytic kernel here.  SURVEY.md section 8f, N2."""
import pytest
import torch

from fixtures import synthetic
from oracle import heads_oracle as HO
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
REQ = ['sdf_eikonal_loss', 'sdf_distance_loss', 'total_variation_loss', 'entropy_loss']
rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-20)).item()


def _leaves(scene, dtype=torch.float32):
    return {k: scene[k].detach().to(dtype).clone().requires_grad_()
            for k in ('planes', 'w1', 'b1', 'w2', 'b2', 'beta')}


@pytest.mark.parametrize('R,N', [(32, 1000), (64, 4097)])
def test_sdf_and_its_gradient(cuda_lib, R, N):
    from nerf_from_image_b200.heads import sdf_points
    B = 2
    scene, _ = Hh.make_case('p3d_plain', seed=9, batch=B, plane_res=R, device='cuda')
    g = torch.Generator().manual_seed(1)
    pts = ((torch.rand(B, N, 3, generator=g) * 2 - 1) * scene['scene_range']).cuda()
    d, grad = sdf_points(scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'], pts,
                         scene['scene_range'])
    x = pts.double().requires_grad_()
    sd = {k: scene[k].double() for k in ('planes', 'w1', 'b1', 'w2', 'b2')}
    d64 = HO.decoder_first_output(sd['planes'], sd['w1'], sd['b1'], sd['w2'], sd['b2'],
                                  x / scene['scene_range'])
    g64, = torch.autograd.grad(d64.sum(), x)
    assert rel(d, d64) < 1e-5
    assert rel(grad, g64) < 1e-5


@pytest.mark.parametrize('layout', ['channel_first', 'channel_last'])
def test_backward_of_both_outputs(cuda_lib, layout):
    """Gradients of an arbitrary function of (d, grad d) w.r.t. planes and decoder: the second
    one is the reference's double backward (generator.py:538-545)."""
    from nerf_from_image_b200.heads import sdf_points
    B, R, N = 2, 32, 3000
    scene, _ = Hh.make_case('p3d_plain', seed=4, batch=B, plane_res=R, device='cuda')
    g = torch.Generator().manual_seed(2)
    pts = ((torch.rand(B, N, 3, generator=g) * 2 - 1) * scene['scene_range']).cuda()
    wd = torch.randn(B, N, generator=g).cuda()
    wg = torch.randn(B, N, 3, generator=g).cuda()
    # ground truth in float64 through the oracle's twice-differentiable fetch
    L64 = _leaves(scene, torch.float64)
    x = pts.double().requires_grad_()
    d64 = HO.decoder_first_output(L64['planes'], L64['w1'], L64['b1'], L64['w2'], L64['b2'],
                                  x / scene['scene_range'])
    g64, = torch.autograd.grad(d64.sum(), x, create_graph=True)
    loss64 = (d64 * wd.double()).sum() + (g64 * wg.double()).sum() + (g64.norm(dim=-1) - 1).square().sum()
    names = ['planes', 'w1', 'b1', 'w2', 'b2']
    ref = torch.autograd.grad(loss64, [L64[n] for n in names])
    L = _leaves(scene)
    planes = L['planes'].permute(0, 1, 3, 4, 2).contiguous().detach().requires_grad_() \
        if layout == 'channel_last' else L['planes']
    d, gr = sdf_points(planes, L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'], layout)
    loss = (d * wd).sum() + (gr * wg).sum() + (gr.norm(dim=-1) - 1).square().sum()
    got = torch.autograd.grad(loss, [planes] + [L[n] for n in names[1:]])
    gp = got[0].permute(0, 1, 4, 2, 3) if layout == 'channel_last' else got[0]
    assert rel(gp, ref[0]) < 1e-4, rel(gp, ref[0])
    for n, a, b in zip(names[1:], got[1:], ref[1:]):
        if n in ('w2', 'b2'):   # only the SDF row of the last layer is involved
            assert a[1:].abs().max().item() == 0
            a, b = a[:1], b[:1]
        assert rel(a, b) < 1e-4, (n, rel(a, b))


def test_regulariser_heads_match_the_oracle(cuda_lib):
    """The four losses and their gradients, with the reference's two random draws replayed."""
    from nerf_from_image_b200.heads import regulariser_heads
    B, R, nstrata = 2, 32, 32
    scene, _ = Hh.make_case('p3d_plain', seed=3, batch=B, plane_res=R, device='cuda')
    L = _leaves(scene)
    torch.manual_seed(11)
    got = regulariser_heads(L['planes'], L['w1'], L['b1'], L['w2'], L['b2'], L['beta'],
                            scene['scene_range'], REQ)
    state = torch.cuda.get_rng_state()
    torch.manual_seed(11)
    n = nstrata - 1
    noise = torch.rand(B, n, n, n, 3, device='cuda')
    perturb = torch.randn(B, 1, n ** 3, 3, device='cuda').view(B, n ** 3, 3)
    assert torch.equal(state, torch.cuda.get_rng_state())   # same RNG consumption
    L2 = _leaves(scene, torch.float64)
    pts = HO.stratified_points(B, nstrata, scene['scene_range'], noise.double())
    ref = HO.heads(L2['planes'], L2['w1'], L2['b1'], L2['w2'], L2['b2'], L2['beta'],
                   scene['scene_range'], pts, REQ, perturb.double())
    wts = [1.0, 0.1, 3.0, 0.5]
    for k in REQ:
        assert got[k].shape == (B,)
        assert rel(got[k], ref[k]) < 1e-4, (k, rel(got[k], ref[k]))
    names = ['planes', 'w1', 'b1', 'w2', 'b2', 'beta']
    ga = torch.autograd.grad(sum(w * got[k].sum() for w, k in zip(wts, REQ)), [L[n] for n in names])
    gb = torch.autograd.grad(sum(w * ref[k].sum() for w, k in zip(wts, REQ)), [L2[n] for n in names])
    for nme, a, b in zip(names, ga, gb):
        if nme in ('w2', 'b2'):
            a, b = a[:1], b[:1]
        assert rel(a, b) < 2e-4, (nme, rel(a, b))
