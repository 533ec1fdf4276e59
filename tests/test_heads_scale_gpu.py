"""The regulariser heads' SDF point kernels (sdf_points_fwd_kernel / sdf_points_bwd_kernel,
csrc/nfi_heads.cu) at training scale and on the faces of the cube, against float64 oracles.

1. Scale.  The kernels run a persistent grid (nfi_heads.cu::grid_for): one warp per unit of 32
   points, at most 592 CTAs of 4 warps on any device, and each warp strides over the units.  Across
   its units the backward carries per-lane decoder-gradient accumulators and reuses its warp's
   F/G/T/P/V shared-memory rows.  That only matters once a warp owns two units or more, which
   test_heads_gpu.py never reaches (B = 2 of 31^3 points is 1,862 units on 2,368 warps).  The tests
   here pick the batch so that every warp owns two units or more and warps own unequal numbers of
   units, at the training plane resolution 256^2 (and 64^2): sdf_points forward and backward of
   each output alone and of both, the batch against each image alone at B = 32 (the generator
   step's 12-13 units per warp), and regulariser_heads against oracle/heads_oracle.py.
2. Faces.  The heads' reference fetch (lib/ops.py grid_sample2d) clamps the tap indices, not the
   coordinate, so its derivative along an axis flows on [0, R-1): on the lower faces of the cube
   too, not on the upper ones.  The render and the sampler follow F.grid_sample, which is zero on
   both.  Crafted fp32 points on faces, edges and corners pin both rules.

The float64 oracles see each point at the texel coordinates the kernels compute for it in fp32
(texel_exact).  Two discontinuities would otherwise turn fp32 rounding of the INPUT into O(1)
differences at single points: the cell of the bilinear fetch, whose derivative g jumps across texel
boundaries (at 256^2 some of the 238,328 points of B = 8 lie within fp32 rounding of one: against
plain float64 points the eikonal plane gradient is off by 2.7e-3, for the kernel and for the oracle
run in fp32 alike), and the faces (divided by the Python float 1.4 rather than by 1.4f, the point
-1.4f lands at -0.99999998, never on the face).
"""
import itertools
import types

import numpy as np
import pytest
import torch

from oracle import heads_oracle as HO
from oracle import render_oracle as O
from tests import helpers as Hh

pytestmark = pytest.mark.gpu

REQ = ['sdf_eikonal_loss', 'sdf_distance_loss', 'total_variation_loss', 'entropy_loss']
NSTRATA = 32
N_PTS = (NSTRATA - 1) ** 3      # 29,791 = 930 * 32 + 31: each image's last unit is ragged
NAMES = ['planes', 'w1', 'b1', 'w2', 'b2']
# The bars of test_heads_gpu.py.  Measured on an H100 (80 GB HBM3, 700 W), 64^2 and 256^2 alike:
# d and g <= 4.9e-7 rel-L2, the plane and decoder gradients of either output or both <= 1.4e-6;
# regulariser_heads at 256^2 losses <= 5.4e-7, gradients <= 2.9e-6 (beta).
VAL_BAR, GRAD_BAR = 1e-5, 1e-4


@pytest.fixture(scope='module')
def lib(cuda_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return cuda_lib


def launch(B, N):
    """(units, warps) of nfi_heads.cu::grid_for: one unit = 32 points of one image, CTAs of 4 warps,
    at most 148 * 4 CTAs whatever the device."""
    units = -(-N // 32) * B
    return units, min(-(-units // 4), 148 * 4) * 4


def assert_multi_unit(B, N, what):
    units, warps = launch(B, N)
    lo, hi = units // warps, -(-units // warps)
    print('\n%s: %d units on %d warps, %d..%d units per warp' % (what, units, warps, lo, hi))
    assert units >= 2 * warps and units % warps != 0, (units, warps)
    assert lo >= 2 and hi > lo


def rel(a, b):
    return Hh.rel_l2(a.double(), b.double())


def leaves(scene, dtype=torch.float32):
    return {k: scene[k].detach().to(dtype).clone().requires_grad_()
            for k in ('planes', 'w1', 'b1', 'w2', 'b2', 'beta')}


def texel_exact(pts, R, sr32):
    """float64 world points whose float64 texel coordinates are exactly the fp32 ones the kernels
    (and the reference run in fp32) compute for the fp32 points ``pts``: x = p / sr32, then
    ((x + 1) / 2) * (R - 1), each step rounded to fp32.  On the faces that is 0 or R-1 exactly."""
    m = np.float32(R - 1)
    seen = pts.cpu().numpy() / sr32     # IEEE division, as the kernels' p.points[i] / p.scene_range
    ix = ((seen + np.float32(1)) / np.float32(2)) * m
    c64 = ix.astype(np.float64) / float(m) * 2 - 1
    return torch.from_numpy(c64 * float(sr32)).to(pts.device)


def stratified(B, scene_range, seed):
    """fp32 stratified points as regulariser_heads draws them (same arithmetic), seeded."""
    n = NSTRATA - 1
    noise = torch.rand(B, n, n, n, 3, generator=torch.Generator().manual_seed(seed))
    return HO.stratified_points(B, NSTRATA, scene_range, noise).cuda()


def upstream(shape, seed):
    """Upstream weights of d (positive: under zero-mean weights the sums over points behind the b1
    and b2 gradients cancel, b2's = sum wd to ~1/sqrt(N), and fp32 rounding of the sum, in any
    order, shows amplified) and of g."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(shape, generator=g).cuda() + 0.5, torch.randn(shape + (3,), generator=g).cuda()


def loss_d(d, wd):
    return (d * wd).sum()


def loss_g(g, wg):
    """The eikonal term and an arbitrary linear one."""
    return (g * wg).sum() + (g.norm(dim=-1) - 1).square().sum()


def oracle(L64, x64, sr):
    """float64 (d, dd/dx) at world points x64 (a leaf), through the oracle's twice-differentiable
    fetch; ``sr`` the fp32 scene range as a float."""
    d = HO.decoder_first_output(L64['planes'], L64['w1'], L64['b1'], L64['w2'], L64['b2'], x64 / sr)
    g, = torch.autograd.grad(d.sum(), x64, create_graph=True)
    return d, g


def oracle_grads(L64, loss, retain=False):
    """Gradients to NAMES (zero for b2 where the loss depends on g alone)."""
    gs = torch.autograd.grad(loss, [L64[n] for n in NAMES], retain_graph=retain, allow_unused=True)
    return {n: torch.zeros_like(L64[n]) if x is None else x for n, x in zip(NAMES, gs)}


def kernel_backward(L, pts, sr, g_d, g_g):
    """SdfPoints.backward called directly, so that an output without upstream reaches the kernel as
    NULL (autograd hands a Function zeros for an unused output): g_d == NULL / g_grad == NULL."""
    from nerf_from_image_b200.fused import planes_to_channel_last
    from nerf_from_image_b200.heads import SdfPoints
    f32 = lambda t: t.detach().float().contiguous()
    ctx = types.SimpleNamespace(
        saved_tensors=(planes_to_channel_last(L['planes'].detach()), f32(L['w1']), f32(L['b1']),
                       f32(L['w2']), f32(L['b2']), f32(pts)),
        needs_input_grad=(True,) * 5 + (False,) * 4, scene_range=float(sr), layout='channel_first')
    return dict(zip(NAMES, SdfPoints.backward(ctx, g_d, g_g)[:5]))


def grad_errors(got, ref, what):
    """rel-L2 per parameter; rows 1.. of w2 / b2 (the colour outputs) must get exactly zero."""
    errs = {}
    for n in NAMES:
        a, b = got[n], ref[n]
        if n in ('w2', 'b2'):
            assert a[1:].abs().max().item() == 0, (what, n)
            a, b = a[:1], b[:1]
        errs[n] = rel(a, b)
    print('  %s rel-L2 vs float64: ' % what + ', '.join('%s %.2e' % kv for kv in errs.items()))
    return errs


# ================================================================ 1. scale

@pytest.mark.parametrize('layout', ['channel_first', 'channel_last'])
@pytest.mark.parametrize('R', [64, 256])
def test_sdf_points_against_float64(lib, R, layout):
    """d and g, and the gradients to planes and decoder of a loss of both outputs, of d alone and of
    g alone (the kernel's g_grad == NULL and g_d == NULL paths)."""
    from nerf_from_image_b200.heads import sdf_points
    B = 6
    assert_multi_unit(B, N_PTS, 'sdf_points R=%d B=%d' % (R, B))
    scene, _ = Hh.make_case('p3d_plain', seed=21, batch=B, plane_res=R, device='cuda')
    sr32 = np.float32(scene['scene_range'])
    sr = float(sr32)
    pts = stratified(B, scene['scene_range'], seed=R)
    wd, wg = upstream((B, N_PTS), R + 1)
    L64 = leaves(scene, torch.float64)
    d64, g64 = oracle(L64, texel_exact(pts, R, sr32).requires_grad_(), sr)
    ref_d = oracle_grads(L64, loss_d(d64, wd.double()), retain=True)
    ref_g = oracle_grads(L64, loss_g(g64, wg.double()))
    ref_both = {n: ref_d[n] + ref_g[n] for n in NAMES}

    L = leaves(scene)
    planes = L['planes'].permute(0, 1, 3, 4, 2).contiguous().detach().requires_grad_() \
        if layout == 'channel_last' else L['planes']
    d, g = sdf_points(planes, L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'], layout)
    vals = {'d': rel(d, d64), 'g': rel(g, g64)}
    print('  values rel-L2 vs float64: d %.2e, g %.2e' % (vals['d'], vals['g']))
    assert max(vals.values()) < VAL_BAR, vals
    got = torch.autograd.grad(loss_d(d, wd) + loss_g(g, wg), [planes] + [L[n] for n in NAMES[1:]])
    got = dict(zip(NAMES, got))
    if layout == 'channel_last':
        got['planes'] = got['planes'].permute(0, 1, 4, 2, 3)
    errs = grad_errors(got, ref_both, 'both outputs')
    # each output alone, with the upstream gradient the loss above sends it
    gl = g.detach().requires_grad_()
    g_up, = torch.autograd.grad(loss_g(gl, wg), gl)
    errs_d = grad_errors(kernel_backward(L, pts, sr, wd, None), ref_d, 'd alone')
    errs_g = grad_errors(kernel_backward(L, pts, sr, None, g_up), ref_g, 'g alone')
    for e in (errs, errs_d, errs_g):
        assert max(e.values()) < GRAD_BAR, e


def test_batch_equals_each_image_alone(lib):
    """The generator step's 32 images at 256^2 (12-13 units per warp) against each image run alone
    (1 unit per warp): d and g bit for bit (no arithmetic crosses points), each image's plane
    gradient up to the order of its atomics, the decoder gradients the sum over the images."""
    from nerf_from_image_b200.heads import sdf_points
    B, R = 32, 256
    assert_multi_unit(B, N_PTS, 'sdf_points batch R=%d B=%d' % (R, B))
    assert launch(1, N_PTS)[0] <= launch(1, N_PTS)[1]
    scene, _ = Hh.make_case('p3d_plain', seed=23, batch=B, plane_res=R, device='cuda')
    pts = stratified(B, scene['scene_range'], seed=5)
    wd, wg = upstream((B, N_PTS), 6)
    L = leaves(scene)
    d, g = sdf_points(L['planes'], L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'])
    got = dict(zip(NAMES, torch.autograd.grad(loss_d(d, wd) + loss_g(g, wg), [L[n] for n in NAMES])))
    total = None
    worst = 0.0
    for b in range(B):
        Lb = {k: (v[b:b + 1] if k == 'planes' else v).detach().clone().requires_grad_()
              for k, v in L.items()}
        db, gb = sdf_points(Lb['planes'], Lb['w1'], Lb['b1'], Lb['w2'], Lb['b2'], pts[b:b + 1],
                            scene['scene_range'])
        assert torch.equal(db[0], d[b]) and torch.equal(gb[0], g[b]), b
        gr = torch.autograd.grad(loss_d(db, wd[b:b + 1]) + loss_g(gb, wg[b:b + 1]),
                                 [Lb[n] for n in NAMES])
        e = rel(got['planes'][b], gr[0][0])
        worst = max(worst, e)
        assert e < 1e-5, (b, e)
        total = list(gr[1:]) if total is None else [t + x for t, x in zip(total, gr[1:])]
    errs = {n: rel(got[n], t) for n, t in zip(NAMES[1:], total)}
    print('  batch vs alone rel-L2: planes (worst image) %.2e, ' % worst
          + ', '.join('%s %.2e' % kv for kv in errs.items()))
    assert max(errs.values()) < 1e-4, errs


# The TV head's |t(d) - t(d2)| has no derivative where the two values meet, and a point whose
# difference is within fp32 rounding of zero can take the other branch in fp32 (the oracle run in
# fp32 does so at 9 of 238,328 points).  Where float64's difference is under TV_TAU, far above the
# kernels' rounding of it, the oracle takes the sign of the kernels' own difference.
TV_TAU = 1e-5


def tv_terms(d, d2, beta, use_sdf):
    """The TV head's per-point difference (heads_oracle.heads)."""
    if use_sdf:
        return HO.laplace_cdf(-d, beta) - HO.laplace_cdf(-d2, beta)
    return torch.sigmoid(d - 1) - torch.sigmoid(d2 - 1)


def tv_on_the_kernels_branches(L, L2, layout, planes, scene_range, pts, pts2, x64, x2_64, sr,
                               use_sdf):
    """float64 TV loss [B] at the points x64 and perturbed points x2_64, on the kernels' branch of
    |.| near zero; and the number of points whose branch differs from float64's."""
    from nerf_from_image_b200.heads import sdf_points
    with torch.no_grad():
        dk = [sdf_points(planes, L['w1'], L['b1'], L['w2'], L['b2'], p, scene_range, layout,
                         want_grad=False)[0] for p in (pts, pts2)]
        tk = tv_terms(dk[0], dk[1], L['beta'], use_sdf)
    dec = lambda x: HO.decoder_first_output(L2['planes'], L2['w1'], L2['b1'], L2['w2'], L2['b2'],
                                            x / sr)
    t64 = tv_terms(dec(x64), dec(x2_64), L2['beta'], use_sdf)
    near = t64.detach().abs() < TV_TAU
    s = torch.where(near, tk.sign().double(), t64.detach().sign())
    # (where both Laplace CDFs saturate, fp32's difference is 0: sign 0, no gradient, as in fp32)
    return (s * t64).mean(dim=1), int((s * t64.detach().sign() < 0).sum())


@pytest.mark.parametrize('layout,use_sdf', [('channel_first', True), ('channel_last', True),
                                            ('channel_first', False)],
                         ids=['sdf-channel_first', 'sdf-channel_last', 'density-channel_first'])
def test_regulariser_heads_at_training_scale(lib, layout, use_sdf):
    """The four losses (the sigmoid TV and entropy pair without an SDF) and their gradients to planes,
    decoder and beta, with the two random draws replayed, at 256^2 and B = 8."""
    from nerf_from_image_b200.heads import regulariser_heads
    B, R = 8, 256
    assert_multi_unit(B, N_PTS, 'regulariser_heads R=%d B=%d %s' % (R, B, layout))
    req = REQ if use_sdf else ['total_variation_loss', 'entropy_loss']
    scene, _ = Hh.make_case('p3d_plain', seed=3, batch=B, plane_res=R, device='cuda')
    sr32 = np.float32(scene['scene_range'])
    sr = float(sr32)
    L = leaves(scene)
    planes = L['planes'].permute(0, 1, 3, 4, 2).contiguous().detach().requires_grad_() \
        if layout == 'channel_last' else L['planes']
    torch.manual_seed(11)
    got = regulariser_heads(planes, L['w1'], L['b1'], L['w2'], L['b2'], L['beta'],
                            scene['scene_range'], req, use_sdf=use_sdf, layout=layout)
    state = torch.cuda.get_rng_state()
    torch.manual_seed(11)
    n = NSTRATA - 1
    noise = torch.rand(B, n, n, n, 3, device='cuda')
    perturb = torch.randn(B, 1, n ** 3, 3, device='cuda').view(B, n ** 3, 3)
    assert torch.equal(state, torch.cuda.get_rng_state())   # same RNG consumption
    # the kernels' fp32 points and perturbed points, computed as regulariser_heads computes them
    pts = HO.stratified_points(B, NSTRATA, scene['scene_range'], noise)
    coords = (pts / scene['scene_range']).view(B, 1, -1, 3)
    pts2 = (coords + perturb.view(B, 1, -1, 3) * 0.004).view(B, -1, 3) * scene['scene_range']
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    L2 = leaves(scene, torch.float64)
    x64, x2_64 = texel_exact(pts, R, sr32), texel_exact(pts2, R, sr32)
    ref = HO.heads(L2['planes'], L2['w1'], L2['b1'], L2['w2'], L2['b2'], L2['beta'], sr, x64,
                   [k for k in req if k != 'total_variation_loss'], use_sdf=use_sdf)
    ref['total_variation_loss'], flipped = tv_on_the_kernels_branches(
        L, L2, layout, planes, scene['scene_range'], pts, pts2, x64, x2_64, sr, use_sdf)
    names = NAMES + (['beta'] if use_sdf else [])
    wts = [1.0, 0.1, 3.0, 0.5][-len(req):]
    gb = torch.autograd.grad(sum(w * ref[k].sum() for w, k in zip(wts, req)), [L2[n] for n in names])
    torch.cuda.synchronize()
    print('  float64 oracle: %.2f GB above the %.2f GB held before it; the kernel\'s TV branch '
          'differs at %d of %d points' % ((torch.cuda.max_memory_allocated() - base) / 2 ** 30,
                                          base / 2 ** 30, flipped, B * N_PTS))
    assert flipped <= 1e-4 * B * N_PTS
    errs = {k: rel(got[k], ref[k]) for k in req}
    ga = torch.autograd.grad(sum(w * got[k].sum() for w, k in zip(wts, req)),
                             [planes] + [L[n] for n in names[1:]])
    ga = list(ga)
    if layout == 'channel_last':
        ga[0] = ga[0].permute(0, 1, 4, 2, 3)
    for nme, a, b in zip(names, ga, gb):
        if nme in ('w2', 'b2'):
            assert a[1:].abs().max().item() == 0, nme
            a, b = a[:1], b[:1]
        errs['grad_' + nme] = rel(a, b)
    print('  rel-L2 vs float64: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    for k, e in errs.items():
        assert e < (1e-4 if k in req else 2e-4), (k, e)


# ================================================================ 2. faces

# Coordinates (normalised, x / scene_range) put on one, two or three axes of a point.  In fp32,
# (1 - 2^-24) + 1 rounds to 2 (a tie, to even), so texel coordinate R-1: on the upper face for the
# kernels and for the reference run in fp32.  1 - 2^-22 stays inside, and unlike 1 - 2^-23 a point
# of the p3d scene range (1.4f) divides to it.
FACE_VALUES = {'lower': -1.0, 'lower_in': -1 + 2 ** -24, 'upper_in': 1 - 2 ** -22,
               'upper_fp32': 1 - 2 ** -24, 'upper': 1.0}
FACE_KINDS = list(FACE_VALUES) + ['mixed']
B_FACE, REP = 2, 16


def face_coords(kind, n_axes, seed):
    """[B, N, 3] fp32 coordinates: for every choice of n_axes axes (faces, edges, corners) and of
    face values on them (every value of FACE_VALUES under 'mixed'), REP points with the other axes
    drawn inside the cube.  Also returns the mask of the face-valued entries."""
    g = torch.Generator().manual_seed(seed)
    vals = list(FACE_VALUES.values()) if kind == 'mixed' else [FACE_VALUES[kind]]
    rows, masks = [], []
    for axes in itertools.combinations(range(3), n_axes):
        for combo in itertools.product(vals, repeat=n_axes):
            c = torch.rand(B_FACE, REP, 3, generator=g) * 1.8 - 0.9
            m = torch.zeros(B_FACE, REP, 3, dtype=torch.bool)
            for a, v in zip(axes, combo):
                c[..., a], m[..., a] = v, True
            rows.append(c)
            masks.append(m)
    return torch.cat(rows, 1), torch.cat(masks, 1)


def outside_coords(seed, n=512):
    """Points up to 1.02 outside the cube, each outside along at least one axis."""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(B_FACE, n, 3, generator=g) * 2.04 - 1.02
    ax = torch.randint(0, 3, (B_FACE, n), generator=g)
    far = torch.where(torch.rand(B_FACE, n, generator=g) < 0.5, -1.0, 1.0) * \
        (1 + 0.02 * torch.rand(B_FACE, n, generator=g).clamp_min(1e-3))
    c.scatter_(2, ax[..., None], far[..., None])
    return c


def world_points(c, mask, sr32):
    """fp32 world points c * sr32 whose coordinate as the kernels compute it (fp32 division by
    sr32) is c wherever ``mask`` is set."""
    c32, mask = c.numpy().astype(np.float32), mask.numpy()
    pts = c32 * sr32
    bad = mask & (pts / sr32 != c32)   # where the rounded product does not divide back: a neighbour
    for d in (np.inf, -np.inf):
        nb = np.nextafter(pts, np.float32(d))
        fix = bad & (nb / sr32 == c32)
        pts[fix], bad = nb[fix], bad & ~fix
    assert ((pts / sr32)[mask] == c32[mask]).all()
    return torch.from_numpy(pts)


def face_case(kind, n_axes, R, seed):
    """Scene, fp32 scene range as a float, the kernels' fp32 points and the oracle's float64 ones."""
    scene, _ = Hh.make_case('p3d_plain', seed=seed, batch=B_FACE, plane_res=R, device='cuda')
    sr32 = np.float32(scene['scene_range'])
    if kind == 'outside':
        c = outside_coords(seed)
        mask = torch.zeros_like(c, dtype=torch.bool)
    else:
        c, mask = face_coords(kind, n_axes, seed)
    pts = world_points(c, mask, sr32).cuda()
    return scene, float(sr32), pts, texel_exact(pts, R, sr32)


FACE_CASES = [(k, n) for k in FACE_KINDS for n in (1, 2, 3)]
face_ids = ['%s-%s' % (k, ('face', 'edge', 'corner')[n - 1]) for k, n in FACE_CASES]


@pytest.mark.parametrize('R', [64, 256])
@pytest.mark.parametrize('kind,n_axes', FACE_CASES, ids=face_ids)
def test_sdf_points_on_the_faces(lib, kind, n_axes, R):
    """d, g and the backward of both outputs at points on the faces, edges and corners, against the
    heads' reference fetch in float64: the derivative along an axis flows at texel coordinate 0 and
    is zero at R-1."""
    from nerf_from_image_b200.heads import sdf_points
    scene, sr, pts, x64 = face_case(kind, n_axes, R, seed=31 + n_axes)
    N = pts.shape[1]
    wd, wg = upstream((B_FACE, N), 7)
    L64 = leaves(scene, torch.float64)
    d64, g64 = oracle(L64, x64.requires_grad_(), sr)
    ref = oracle_grads(L64, loss_d(d64, wd.double()) + loss_g(g64, wg.double()))
    L = leaves(scene)
    d, g = sdf_points(L['planes'], L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'])
    vals = {'d': rel(d, d64), 'g': rel(g, g64)}
    print('\n  %d points, values rel-L2 vs float64: d %.2e, g %.2e' % (B_FACE * N, vals['d'], vals['g']))
    got = dict(zip(NAMES, torch.autograd.grad(loss_d(d, wd) + loss_g(g, wg), [L[n] for n in NAMES])))
    errs = grad_errors(got, ref, 'both outputs')
    assert max(vals.values()) < VAL_BAR, vals
    assert max(errs.values()) < GRAD_BAR, errs


@pytest.mark.parametrize('R', [64, 256])
def test_sdf_points_outside_the_cube(lib, R):
    """Points up to 1.02 outside (the TV head's perturbed points): d and g, and the gradients of a
    loss of d alone through a launch without g (the TV head's)."""
    from nerf_from_image_b200.heads import sdf_points
    scene, sr, pts, x64 = face_case('outside', 0, R, seed=41)
    wd, _ = upstream(tuple(pts.shape[:2]), 8)
    L64 = leaves(scene, torch.float64)
    d64, g64 = oracle(L64, x64.requires_grad_(), sr)
    ref = oracle_grads(L64, loss_d(d64, wd.double()))
    L = leaves(scene)
    _, g = sdf_points(L['planes'], L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'])
    d, _ = sdf_points(L['planes'], L['w1'], L['b1'], L['w2'], L['b2'], pts, scene['scene_range'],
                      want_grad=False)
    vals = {'d': rel(d, d64), 'g': rel(g, g64)}
    print('\n  values rel-L2 vs float64: d %.2e, g %.2e' % (vals['d'], vals['g']))
    got = dict(zip(NAMES, torch.autograd.grad(loss_d(d, wd), [L[n] for n in NAMES])))
    errs = grad_errors(got, ref, 'd alone')
    assert max(vals.values()) < VAL_BAR, vals
    assert max(errs.values()) < GRAD_BAR, errs


@pytest.mark.parametrize('kind,n_axes', FACE_CASES + [('outside', 0)],
                         ids=face_ids + ['outside'])
def test_sampler_normals_on_the_faces(lib, kind, n_axes):
    """The sampler's normals at the same points follow F.grid_sample's rule (zero derivative along
    an axis on both of its faces), against O.sampler in float64: the heads' rule stays out of the
    render and sampler path."""
    from nerf_from_image_b200.sampler import FusedSampler
    R = 256
    scene, sr, pts, x64 = face_case(kind, n_axes, R, seed=51 + n_axes)
    req = ['sdf_distance', 'normals']
    ref = O.sampler(x64, *[scene[k].double() for k in ('planes', 'w1', 'b1', 'w2', 'b2', 'palette',
                                                         'beta', 'alpha')], sr, request=req)
    sampler = FusedSampler(scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'],
                           scene['palette'], scene['beta'], scene['alpha'], scene['scene_range'])
    with torch.no_grad():
        out = sampler(pts, req)
    errs = {k: rel(out[k], ref[k].detach()) for k in req}
    print('\n  sampler rel-L2 vs float64: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    assert errs['sdf_distance'] < VAL_BAR and errs['normals'] < 2e-4, errs
