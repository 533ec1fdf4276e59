"""oracle/heads_oracle.py against the UNMODIFIED reference Generator's regulariser heads
(models/generator.py:520-585; its synthesis network stubbed to return the planes under test),
values and gradients w.r.t. planes / decoder / beta, with the same random draws.  The reference
runs live where it is installed, its recorded output stands in elsewhere
(tests.helpers.reference_output)."""
import torch

from oracle import heads_oracle as HO
from oracle import reference_lift as RL
from tests import helpers as Hh

REQ = ['sdf_eikonal_loss', 'sdf_distance_loss', 'total_variation_loss', 'entropy_loss']


def _run_reference(scene, B, R):
    """The reference Generator's four heads under torch.manual_seed(11): (losses, effective
    decoder weights and beta, gradients to planes / raw weights / beta, the weight gains)."""
    g = RL.build_reference_generator(scene)
    g.train()   # the eikonal head asserts self.training (generator.py:531)
    planes = scene['planes'].clone().requires_grad_()
    g.synthesis_network.planes = planes.reshape(B, 96, R, R)
    ws = torch.zeros(B, 15, 512)
    torch.manual_seed(11)
    ref = g(None, ws, request_model_outputs=REQ, model_inputs={'attention_values': scene['palette']})
    l1, l2 = g.decoder.net[0], g.decoder.net[2]
    eff = dict(w1=l1.weight * l1.weight_gain, b1=l1.bias * l1.bias_gain,
               w2=l2.weight * l2.weight_gain, b2=l2.bias * l2.bias_gain, beta=g.beta.clone())
    wts = torch.tensor([1.0, 0.1, 3.0, 0.5])
    loss_r = sum(w * ref[k].sum() for w, k in zip(wts, REQ))
    gr = torch.autograd.grad(loss_r, [planes, l1.weight, l2.weight, g.beta])
    gains = torch.tensor([l1.weight_gain, l2.weight_gain])
    return {k: ref[k] for k in REQ}, eff, list(gr), gains


def _check_oracle(scene, B, nstrata, noise, perturb, ref, eff, gr, gains):
    leaves = {k: v.detach().clone().requires_grad_() for k, v in eff.items()}
    planes2 = scene['planes'].clone().requires_grad_()
    pts = HO.stratified_points(B, nstrata, scene['scene_range'], noise)
    got = HO.heads(planes2, leaves['w1'], leaves['b1'], leaves['w2'], leaves['b2'], leaves['beta'],
                   scene['scene_range'], pts, REQ, perturb)
    for k in REQ:
        assert got[k].shape == ref[k].shape == (B,)
        assert (got[k] - ref[k]).abs().max().item() < 2e-5 * max(1.0, ref[k].abs().max().item()), k
    wts = torch.tensor([1.0, 0.1, 3.0, 0.5])
    loss_g = sum(w * got[k].sum() for w, k in zip(wts, REQ))
    gg = torch.autograd.grad(loss_g, [planes2, leaves['w1'], leaves['w2'], leaves['beta']])
    rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-12)).item()
    assert rel(gg[0], gr[0]) < 1e-4
    assert rel(gg[1] * gains[0], gr[1]) < 1e-4      # d/d raw weight = gain * d/d effective
    assert rel((gg[2] * gains[1])[:1], gr[2][:1]) < 1e-4
    assert rel(gg[3], gr[3]) < 1e-4


def test_heads_match_the_reference_on_the_faces(request, monkeypatch):
    """The reference's stratified draw (torch.rand_like of lib/ops.py:23) replaced so that the
    first and last stratum of every axis put their points exactly on the cube's lower and upper
    faces (coordinate -1 and +1 after the reference's own division by scene_range), edges and
    corners included: about 18 % of the points.  There the reference's twice-differentiable fetch
    (lib/ops.py grid_sample2d) differentiates along an axis on the lower face and not on the upper
    one, and so must the oracle."""
    B, R, nstrata = 2, 16, 32
    n = nstrata - 1
    scene, _ = Hh.make_case('p3d_plain', seed=5, batch=B, plane_res=R)
    r = torch.arange(n)
    bins = torch.stack(torch.meshgrid(r, r, r, indexing='xy'), dim=-1).expand(B, -1, -1, -1, -1)
    noise = torch.rand(B, n, n, n, 3, generator=torch.Generator().manual_seed(12))
    noise[bins == 0] = 0.0                       # (0 + 0) / 31 * 2 - 1 = -1
    noise[bins == n - 1] = 1 - 2 ** -24          # 30 + (1 - 2^-24) rounds to 31: +1 in fp32
    coords = HO.stratified_points(B, nstrata, scene['scene_range'], noise) / scene['scene_range']
    per_face = B * n * n
    assert ((coords == -1).sum(dim=(0, 1)) == per_face).all()
    assert ((coords == 1).sum(dim=(0, 1)) == per_face).all()
    assert ((coords.abs() == 1).sum(dim=-1) == 3).sum() == 8 * B      # corners

    def reference():
        def rand_like(t, **kw):
            assert t.shape == noise.shape, t.shape
            return noise.clone()
        RL.build_reference_generator(scene)   # its TorchScript functions compile with the real draw
        with monkeypatch.context() as m:
            m.setattr(torch, 'rand_like', rand_like)
            return _run_reference(scene, B, R)

    ref, eff, gr, gains = Hh.reference_output(request, reference)
    # the stratified draw is replaced, so the perturbation is the first draw after the seed
    torch.manual_seed(11)
    perturb = torch.randn(B, 1, n ** 3, 3).view(B, n ** 3, 3)
    _check_oracle(scene, B, nstrata, noise, perturb, ref, eff, gr, gains)


def test_heads_match_the_reference(request):
    B, R, nstrata = 2, 16, 32
    scene, _ = Hh.make_case('p3d_plain', seed=3, batch=B, plane_res=R)
    ref, eff, gr, gains = Hh.reference_output(request, lambda: _run_reference(scene, B, R))
    # replay the two draws: rand_like(bins) (ops.py:23), then randn_like(eik_coords) (:554)
    torch.manual_seed(11)
    n = nstrata - 1
    noise = torch.rand(B, n, n, n, 3)
    perturb = torch.randn(B, 1, n ** 3, 3).view(B, n ** 3, 3)
    _check_oracle(scene, B, nstrata, noise, perturb, ref, eff, gr, gains)
