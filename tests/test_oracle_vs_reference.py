"""Pins the oracle against the reference's own code (CPU).

The reference runs live where it is installed (oracle/_ref); elsewhere its outputs recorded under
tests/golden/reference/ stand in for it (tests.helpers.reference_output).
"""
import pytest
import torch

from oracle import pose_oracle as PO
from oracle import reference_lift as RL
from oracle import render_oracle as O
from tests import helpers as Hh


@pytest.mark.parametrize('case', list(Hh.CASES))
@pytest.mark.parametrize('randomize', [True, False])
def test_render_matches_reference(request, case, randomize):
    scene, cams = Hh.make_case(case, seed=2, batch=2, plane_res=24)
    out, nt, nu = Hh.reference_output(request, lambda: RL.reference_render(
        scene, cams, 12, 20, 12, seed=4, randomize=randomize))
    o = Hh.run_oracle(scene, cams, 12, 20, 12, nt, nu)
    for ref, k in zip(out[:3], ('rgb', 'depth', 'mask')):
        assert (ref - o[k]).abs().max().item() < 2e-5, k


@pytest.mark.parametrize('kw', [dict(fine_sampling=False), dict(use_sdf=False),
                                dict(compute_semantics=True), dict(compute_coords=True),
                                dict(compute_normals=True), dict(force_no_cam_grad=True)])
def test_render_variants_match_reference(request, kw):
    scene, cams = Hh.make_case('p3d_bbox', seed=3, batch=2, plane_res=24)
    out, nt, nu = Hh.reference_output(request, lambda: RL.reference_render(
        scene, cams, 12, 12, 10, seed=5, **kw))
    o = Hh.run_oracle(scene, cams, 12, 12, 10, nt, nu, **kw)
    for ref, k in zip(out[:3], ('rgb', 'depth', 'mask')):
        assert (ref - o[k]).abs().max().item() < 2e-5, k
    if out[3] is not None:
        assert (out[3] - o['normals']).abs().max().item() < 1e-4
    if out[4] is not None:
        assert (out[4] - o['semantics']).abs().max().item() < 2e-5


@pytest.mark.parametrize('case,A,kw', [('p3d_plain', 10, {}), ('chairs_white_center', 0, {}),
                                       ('cub_ortho', 10, dict(compute_semantics=True)),
                                       ('p3d_bbox', 10, dict(force_no_cam_grad=True)),
                                       ('p3d_plain', 10, dict(compute_normals=True))])
def test_view_direction_conditioning_matches_reference(request, case, A, kw):
    """--use_viewdir (run.py:216-221, models/generator.py:189-253,662-663): the reference
    Generator built with use_viewdir=True and given the oracle scene's ViewDirectionMapper
    weights, called by the reference's own render(), against the oracle's restatement of the
    mapper trunk (per ray) and closure (per sample)."""
    from fixtures import synthetic
    scene, cams = Hh.make_case(case, seed=2, batch=2, plane_res=24, attention_values=A)
    scene = synthetic.add_view_mapper(scene)
    out, nt, nu = Hh.reference_output(request, lambda: RL.reference_render(
        scene, cams, 12, 20, 12, seed=4, **kw))
    o = Hh.run_oracle(scene, cams, 12, 20, 12, nt, nu, **kw)
    for ref, k in zip(out[:3], ('rgb', 'depth', 'mask')):
        assert (ref - o[k]).abs().max().item() < 2e-5, k
    if out[3] is not None:
        assert (out[3] - o['normals']).abs().max().item() < 1e-4
    if out[4] is not None:
        assert (out[4] - o['semantics']).abs().max().item() < 2e-5
    # the trunk alone, against the module (bit-identical: same ops in the same order)
    def trunk():
        g = RL.build_reference_generator(scene)
        m, w3, b3 = O.effective_view_mapper_weights(g.viewdir_mapper)
        d = torch.nn.functional.normalize(torch.randn(3, 5, 1, 3), dim=-1)
        closure = g.viewdir_mapper(d)
        x_ref = dict(zip(closure.__code__.co_freevars,
                         (c.cell_contents for c in closure.__closure__)))['x']
        return m, d, x_ref
    m, d, x_ref = Hh.reference_output(request, trunk, '.trunk')
    assert torch.equal(O.view_mapper_trunk(d, m), x_ref)


def test_stage_functions_match_reference(request):
    scene, _ = Hh.make_case('p3d_bbox', seed=6, batch=2)
    cam_cases = ('p3d_bbox', 'cub_ortho_bbox', 'chairs_white_center')
    torch.manual_seed(0)
    w = torch.rand(50, 16)
    bins = torch.sort(torch.rand(50, 15), dim=-1).values

    def reference():
        nerf_utils, _ = RL._import_reference()
        rays = []
        for cam_case in cam_cases:
            _, cams = Hh.make_case(cam_case, seed=6, batch=2)
            ro, rd = nerf_utils.get_ray_bundle(9, 13, cams['focal'], cams['c2w'], cams['bbox'],
                                               cams['center'])
            dn = torch.nn.functional.normalize(rd, dim=-1)
            rays.append((ro, rd) + tuple(nerf_utils.compute_near_far_planes(ro, dn,
                                                                            scene['scene_range'])))
        torch.manual_seed(1)
        s_rand = nerf_utils.sample_pdf(bins, w[..., 1:-1], 16, deterministic=False)
        s_det = nerf_utils.sample_pdf(bins, w[..., 1:-1], 16, deterministic=True)
        return rays, s_rand, s_det

    rays, s_rand, s_det = Hh.reference_output(request, reference)
    for cam_case, (ro, rd, rn, rf) in zip(cam_cases, rays):
        _, cams = Hh.make_case(cam_case, seed=6, batch=2)
        o, d = O.ray_bundle(9, 13, cams['focal'], cams['c2w'], cams['bbox'], cams['center'])
        assert (ro - o).abs().max() < 1e-6 and (rd - d).abs().max() < 1e-6
        dn = torch.nn.functional.normalize(rd, dim=-1)
        n, f, _ = O.near_far_planes(o, dn, scene['scene_range'])
        assert torch.equal(rn, n) and torch.equal(rf, f)
    torch.manual_seed(1)
    u = torch.rand(50, 16)
    assert torch.allclose(s_rand, O.inverse_cdf_samples(bins, w[..., 1:-1], u), atol=1e-6)
    assert torch.allclose(s_det, O.inverse_cdf_samples(bins, w[..., 1:-1],
                                                       O.deterministic_u(16, 50)), atol=1e-6)


def test_missed_rays_do_not_need_the_global_fallback():
    """The CUDA path skips lib/nerf_utils.py:258-259; images must not change."""
    scene, cams = Hh.make_case('p3d_plain', seed=8, batch=2)
    cams['focal'] = torch.tensor([0.35, 0.4])  # wide field of view: corner rays miss the cube
    from fixtures import synthetic
    nt, nu = synthetic.make_noise(1, 2, 16, 16, 8)
    a = Hh.run_oracle(scene, cams, 16, 16, 8, nt, nu, global_near_far_fallback=True)
    b = Hh.run_oracle(scene, cams, 16, 16, 8, nt, nu, global_near_far_fallback=False)
    o, d = O.ray_bundle(16, 16, cams['focal'], cams['c2w'], cams['bbox'], None)
    hit = O.near_far_planes(o, torch.nn.functional.normalize(d, dim=-1), scene['scene_range'])[2]
    assert (~hit).any() and hit.any()
    for k in ('rgb', 'depth', 'mask'):
        assert torch.equal(a[k], b[k]), k


def sampler_points(scene, batch, n, seed):
    """Points filling the cube and a margin outside it (the out-of-box mask must trigger)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(batch, 5, n // 5, 3, generator=g) * 2 - 1) * 1.15 * scene['scene_range']


@pytest.mark.parametrize('A,use_sdf,request_', [
    (10, True, ['sigma', 'rgb']),
    (10, True, ['sdf_distance', 'sigma', 'rgb', 'semantics', 'coords']),
    (0, True, ['sigma', 'rgb', 'sdf_distance']),
    (10, False, ['sigma', 'rgb']),
])
def test_sampler_matches_reference(request, A, use_sdf, request_):
    scene, _ = Hh.make_case('p3d_plain', seed=12, batch=2, plane_res=24, attention_values=A)
    x = sampler_points(scene, 2, 200, 3)
    with torch.no_grad():
        ref = Hh.reference_output(request, lambda: RL.reference_sampler(
            scene, x, request_, use_sdf=use_sdf))
        o = O.sampler(x, scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'],
                      scene['palette'], scene['beta'], scene['alpha'], scene['scene_range'],
                      request=request_, use_sdf=use_sdf)
    assert sorted(ref) == sorted(o)
    for k in ref:
        assert ref[k].shape == o[k].shape, k
        assert (ref[k] - o[k]).abs().max().item() < 2e-5, k


def test_sampler_normals_and_bbox_match_reference(request):
    scene, _ = Hh.make_case('p3d_plain', seed=13, batch=2, plane_res=24)
    x = sampler_points(scene, 2, 200, 4)
    ref = Hh.reference_output(request, lambda: RL.reference_sampler(
        scene, x.clone(), ['normals', 'sigma']))
    o = O.sampler(x, scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'],
                  scene['palette'], scene['beta'], scene['alpha'], scene['scene_range'],
                  request=['normals', 'sigma'])
    assert ref['normals'].shape == o['normals'].shape == x.shape
    assert (ref['normals'] - o['normals']).abs().max().item() < 1e-4
    assert (ref['sigma'] - o['sigma']).abs().max().item() < 2e-5
    with torch.no_grad():
        ref = Hh.reference_output(request, lambda: RL.reference_sampler(
            scene, x, ['sigma', 'coords'], bbox_debug=True), '.bbox')
        o = O.sampler(x, scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'],
                      scene['palette'], scene['beta'], scene['alpha'], scene['scene_range'],
                      request=['sigma', 'coords'], bbox_debug=True)
    assert (ref['sigma'] > 50).any()
    assert (ref['sigma'] - o['sigma']).abs().max().item() < 2e-5


def pose_inputs(seed, batch, persp):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(batch, 4, generator=g), dim=-1)
    t2 = 0.3 * torch.randn(batch, 2, generator=g)
    s = 0.8 + 0.5 * torch.rand(batch, generator=g)
    z0 = 0.5 * torch.randn(batch, generator=g) if persp else None
    return z0, t2, s, q


@pytest.mark.parametrize('persp', [True, False])
@pytest.mark.parametrize('flipped', [True, False])
def test_pose_to_matrix_matches_reference(request, persp, flipped):
    z0, t2, s, q = pose_inputs(5, 6, persp)
    leaves_o = [t.clone().requires_grad_() for t in (z0, t2, s, q) if t is not None]
    args = lambda L: ((L[0], L[1], L[2], L[3]) if persp else (None, L[0], L[1], L[2]))
    g = torch.Generator().manual_seed(9)
    wm = torch.randn(6, 4, 4, generator=g)
    wf = torch.randn(6, generator=g)
    loss = lambda m, f: (m * wm).sum() + ((f * wf).sum() if f is not None else 0)

    def reference():
        pu = RL.reference_pose_utils()
        leaves = [t.clone().requires_grad_() for t in (z0, t2, s, q) if t is not None]
        mat_r, f_r = pu.pose_to_matrix(*args(leaves), flipped)
        return mat_r, f_r, list(torch.autograd.grad(loss(mat_r, f_r), leaves))

    mat_r, f_r, gr = Hh.reference_output(request, reference)
    mat_o, f_o = PO.pose_to_matrix(*args(leaves_o), flipped)
    assert torch.equal(mat_r, mat_o)
    assert (f_r is None) == (f_o is None)
    go = torch.autograd.grad(loss(mat_o, f_o), leaves_o)
    for a, b in zip(gr, go):
        assert (a - b).abs().max().item() < 1e-5
    # (lib/pose_utils.py:72 matrix_to_pose, the reference's inverse, does not run under
    # numpy >= 2 -- np.array(copy=False) -- so the round trip is not checked through it)
    rows = PO.quaternion_rows(q)
    eye = torch.eye(3).expand(6, 3, 3)
    assert (rows @ rows.transpose(-1, -2) - eye).abs().max().item() < 1e-5
