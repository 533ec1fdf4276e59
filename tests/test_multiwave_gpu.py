"""The persistent kernels with more tiles than SMs, against float64 oracles.

Every hot kernel runs a persistent grid of min(tiles, SMs) CTAs, and each CTA steps through tiles
with ``tile += gridDim.x``: render_forward_pipe, render_backward_pipe, render_wgrad_pipe,
render_normals_pipe and the synthesis network's conv_tc_kernel.  What a CTA carries from one tile
to the next -- ring positions and mbarrier parities, the D2 slots, its scratch slab, the
weight-gradient chains (flushed every kWgFlush steps of the CTA's whole run and banked until the
final flush), the TMA producer's stage and phase -- only matters once a CTA owns two tiles or
more.  The other tests stay inside one wave (at most 128 render tiles on 132 SMs), so every test
here picks its batch from the device's SM count such that the tile count is at least twice the SM
count and not a multiple of it: CTAs then own unequal numbers of tiles.  Each test asserts that
and prints the tiles per CTA.

1. the render kernels on a ragged 40x56 image (5 x 4 tiles of 8 x 16 rays, the last tile column
   half outside the image): forward, batch-versus-alone bit equality, the inversion backward and
   the decoder-weight gradients in all three routes, against the oracle in float64 on the GPU;
2. the benchmark's own workloads (configs 2, 3 and 4 of bench.py, inputs restated here);
3. the synthesis convolutions at narrow channels (small reduction lengths, so that the tensor
   core's accumulation error stays far below the bars) over several waves: the forward against
   float64, ws.grad of the batch against each image alone, and ws.grad against float64 (an
   expected failure for now, see SYNTH_GRAD_BAR).
"""
import math

import pytest
import torch

from fixtures import synthetic
from oracle import render_oracle as O
from oracle import synthesis_oracle as SO
from tests import helpers as Hh
from tests import helpers_synth as HS
from tests import synthesis_branch_oracle as BO

pytestmark = pytest.mark.gpu

TOL = 2e-4          # forward bar of test_parity_gpu.py
H, W = 40, 56       # 5 x 4 tiles per image, the last tile column half outside the image


@pytest.fixture(scope='module')
def sms(cuda_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles(B, H, W):
    """Render tiles of 8 rows x 16 columns of rays."""
    return B * math.ceil(H / 8) * math.ceil(W / 16)


def per_cta(n_tiles, sms):
    grid = min(n_tiles, sms)
    return n_tiles // grid, -(-n_tiles // grid)


def assert_multiwave(n_tiles, sms, what):
    lo, hi = per_cta(n_tiles, sms)
    print('\n%s: %d tiles on %d SMs, %d..%d tiles per CTA' % (what, n_tiles, sms, lo, hi))
    assert n_tiles >= 2 * sms and n_tiles % sms != 0, (n_tiles, sms)
    assert lo >= 2 and hi > lo


def ragged_batch(sms):
    """About 2.5 waves of the 40x56 image (17 images = 340 tiles on 132 SMs), never a whole
    number of waves."""
    per_image = tiles(1, H, W)
    B = -(-5 * sms // (2 * per_image))
    while tiles(B, H, W) % sms == 0:
        B += 1
    return B


def dbl(d):
    return {k: (v.double() if torch.is_tensor(v) else v) for k, v in d.items()}


def leaves(scene, cams, names, cam_names):
    sc = {k: (v.detach().clone().requires_grad_() if k in names else v) for k, v in scene.items()}
    cm = {k: (v.detach().clone().requires_grad_() if k in cam_names else v)
          for k, v in cams.items()}
    return sc, cm


def upstream(B, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, H, W, 3, generator=g).cuda(), torch.randn(B, H, W, generator=g).cuda())


def z_fine_of(out):
    """The fine depths FusedTriplaneRender saved for its backward ([B*H*W, S])."""
    fn = out[0].grad_fn
    return dict(zip(fn.saved_names, fn.saved_tensors))['z_fine']


def image(scene, cams, nt, nu, b, H, W):
    """Image b of a batch as a batch of one: scene, cameras and noise."""
    sc = {k: (v[b:b + 1] if k in ('planes', 'palette') and v is not None else v)
          for k, v in scene.items()}
    cm = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cams.items()}
    S = nt.shape[-1]
    nu_b = None if nu is None else nu.view(-1, H * W, nu.shape[-1])[b].contiguous()
    return sc, cm, nt[b:b + 1], nu_b, S


def row_bands(H, W, sms):
    """Row ranges of one image that each fit in one wave (row tiles are bit-exact)."""
    step = max(1, sms // math.ceil(W / 16)) * 8
    return [(r0, min(r0 + step, H)) for r0 in range(0, H, step)]


def render_alone(render, scene, cams, nt, nu, b, H, W, sms):
    """Image b rendered on its own, in row bands of at most one wave each; ``render(sc, cm, h,
    nt, nu, rows)`` -> tuple of outputs [1, h, ...].  Returns the bands' outputs joined along the
    rows (None where an output is None)."""
    from nerf_from_image_b200 import parallel as PAR
    sc, cm, nt_b, nu_b, S = image(scene, cams, nt, nu, b, H, W)
    pieces = []
    for r0, r1 in row_bands(H, W, sms):
        assert tiles(1, r1 - r0, W) <= sms
        nt_r, nu_r = PAR.slice_rows(nt_b, nu_b, 1, H, W, r0, r1)
        pieces.append(render(sc, cm, r1 - r0, nt_r, nu_r, None if (r0, r1) == (0, H) else (r0, H)))
    return [None if p[0] is None else torch.cat(p, dim=1) for p in zip(*pieces)]


# ================================================================ 1. render kernels, ragged shape

S_FWD = 16
# (case, attention values, render options, extra_mode, mlp_mode).  A in {0, 3} -> NOUT_PAD 4,
# 10 -> 12, 15 -> 16; mode 4 the pipelined kernels, 0 auto (also pipelined), 1 the SIMT control.
FWD_CASES = [
    ('p3d_bbox', 10, {}, 0, 4),
    ('cub_ortho', 0, {}, 0, 4),
    ('chairs_white_center', 15, {}, 0, 4),
    ('p3d_bbox', 3, {}, 0, 4),
    ('p3d_bbox', 10, dict(use_sdf=False), 0, 4),
    ('chairs_white_center', 10, dict(fine_sampling=False), 0, 4),
    ('p3d_bbox', 10, {}, 1, 4),
    ('chairs_white_center', 15, {}, 2, 4),
    ('cub_ortho', 10, {}, 0, 0),
    ('p3d_bbox', 10, {}, 0, 1),
]


def _fwd_id(c):
    case, A, kw, ex, mode = c
    return '%s-A%d%s%s-mode%d' % (case, A, ''.join('-' + k for k in kw),
                                  ('', '-coords', '-semantics')[ex], mode)


def _check_forward(sms, case, A, kw, extra_mode, mode, normals=False, seed=3):
    B = ragged_batch(sms)
    assert_multiwave(tiles(B, H, W), sms, '%s A=%d %s extra=%d mode=%d normals=%s'
                     % (case, A, kw, extra_mode, mode, normals))
    scene, cams = Hh.make_case(case, seed=seed, batch=B, plane_res=64, attention_values=A,
                               device='cuda')
    fine = kw.get('fine_sampling', True)
    nt, nu = synthetic.make_noise(seed + 70, B, H, W, S_FWD, fine=fine, device='cuda')
    ref = Hh.run_oracle(dbl(scene), dbl(cams), H, W, S_FWD, nt.double(),
                        nu.double() if nu is not None else None, compute_coords=extra_mode == 1,
                        compute_semantics=extra_mode == 2, compute_normals=normals, **kw)
    # planes requiring grad: the kernel keeps the fine depths for the backward, where they can be read
    sc = dict(scene, planes=scene['planes'].clone().requires_grad_())
    out = Hh.run_cuda(sc, cams, H, W, S_FWD, nt, nu, extra_mode=extra_mode, mlp_mode=mode,
                      compute_normals=normals, **kw)
    errs = {'rgb': Hh.rel_l2(out[0].detach().double(), ref['rgb']),
            'depth': Hh.rel_l2(out[1].double(), ref['depth']),
            'mask': Hh.rel_l2(out[2].detach().double(), ref['mask'])}
    if extra_mode:
        errs['extra'] = Hh.rel_l2(out[3].double(), ref['semantics'].detach())
    if normals:
        errs['normals'] = Hh.rel_l2(out[4].double(), ref['normals'].detach())
    if fine:
        zf = z_fine_of(out).view(B, H, W, S_FWD).double()
        zr = ref['z_fine'].sort(dim=-1).values
        o, d = O.ray_bundle(H, W, dbl(cams)['focal'], dbl(cams)['c2w'], dbl(cams)['bbox'],
                            dbl(cams)['center'])
        hit = O.near_far_planes(o, torch.nn.functional.normalize(d, dim=-1),
                                scene['scene_range'])[2]
        assert hit.any()
        errs['z_fine'] = Hh.rel_l2(zf[hit], zr[hit])
        errs['z_fine_max'] = (zf[hit] - zr[hit]).abs().max().item()
    print('  rel-L2 vs float64: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    for k, e in errs.items():
        assert e < Z_FINE_BARS.get(k, 1e-3 if k == 'normals' else TOL), (k, e)


# The fine depths against float64 over ~38,000 rays, depths up to 6: the inverse CDF moves a sample
# by (CDF error) / (pdf), so single samples in low-density bins move most.  Measured on an H100:
# at most 9.4e-5 (cub_ortho; test_fine_depths_match's 2e-5 holds for its 256 rays of p3d), where
# the oracle's own fp32 run leaves 4.8e-5.  The rel-L2 bar is the one a misplaced tile would break.
Z_FINE_BARS = {'z_fine': 1e-5, 'z_fine_max': 2e-4}


@pytest.mark.parametrize('case,A,kw,extra_mode,mode', FWD_CASES, ids=[_fwd_id(c) for c in FWD_CASES])
def test_forward_against_float64(sms, case, A, kw, extra_mode, mode):
    _check_forward(sms, case, A, kw, extra_mode, mode)


@pytest.mark.parametrize('case,A', [('p3d_bbox', 10), ('chairs_white_center', 15)])
def test_normals_and_semantics_against_float64(sms, case, A):
    """render_normals_pipe after render_forward_pipe (mlp_mode 0 picks both)."""
    _check_forward(sms, case, A, {}, 2, 0, normals=True, seed=5)


@pytest.mark.parametrize('case,A,extra_mode,normals,mode', [
    ('p3d_bbox', 10, 2, True, 0),
    ('cub_ortho', 0, 1, False, 4),
    ('chairs_white_center', 15, 0, False, 4),
])
def test_batch_equals_each_image_alone(sms, case, A, extra_mode, normals, mode):
    """Every image of the multi-wave batch equals the same image rendered in one wave, bit for
    bit: rgb, depth, mask, extra, normals and the fine depths."""
    S = S_FWD
    B = ragged_batch(sms)
    assert_multiwave(tiles(B, H, W), sms, 'batch of %d vs each image alone' % B)
    scene, cams = Hh.make_case(case, seed=9, batch=B, plane_res=64, attention_values=A,
                               device='cuda')
    nt, nu = synthetic.make_noise(79, B, H, W, S, device='cuda')

    def render(sc, cm, h, nt_, nu_, rows):
        from nerf_from_image_b200.fused import RenderConfig, fused_render
        cfg = RenderConfig(scene_range=sc['scene_range'], white_background=sc['white_background'],
                           attention_values=A, mlp_mode=mode)
        planes = sc['planes'].clone().requires_grad_()
        out = fused_render(planes, sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                           sc['beta'], sc['alpha'], cm['c2w'], cm['focal'], cm['center'],
                           cm['bbox'], cfg, h, W, S, nt_, nu_, extra_mode,
                           compute_normals=normals, rows=rows)
        n = planes.shape[0]
        zf = z_fine_of(out).view(n, h, W, S)
        return [x.detach() if x is not None else None for x in out] + [zf.detach()]

    full = render(scene, cams, H, nt, nu, None)
    names = ['rgb', 'depth', 'mask', 'extra'] + (['normals'] if normals else []) + ['z_fine']
    for b in range(B):
        part = render_alone(render, scene, cams, nt, nu, b, H, W, sms)
        for n, x, y in zip(names, part, full):
            if y is None:
                assert x is None
                continue
            assert torch.equal(x[0], y[b]), (b, n, (x[0] - y[b]).abs().max().item())


@pytest.mark.parametrize('case,mode,cam_grad', [
    ('p3d_bbox', 4, True), ('cub_ortho', 4, True), ('chairs_white_center', 4, True),
    ('p3d_bbox', 4, False), ('chairs_white_center', 1, True)])
def test_inversion_backward_against_float64(sms, case, mode, cam_grad):
    """render_backward_pipe (decoder frozen): planes, palette, beta, alpha and the cameras."""
    S = S_FWD
    B = ragged_batch(sms)
    assert_multiwave(tiles(B, H, W), sms, 'inversion backward %s mode %d cam_grad %s'
                     % (case, mode, cam_grad))
    scene, cams = Hh.make_case(case, seed=11, batch=B, plane_res=64, device='cuda')
    nt, nu = synthetic.make_noise(81, B, H, W, S, device='cuda')
    names = ['planes', 'palette', 'beta', 'alpha']
    cam_names = [k for k in ('c2w', 'focal', 'bbox', 'center') if cams[k] is not None]
    wr, wm = upstream(B, H, W)
    sc, cm = leaves(dbl(scene), dbl(cams), names, cam_names)
    ref = Hh.run_oracle(sc, cm, H, W, S, nt.double(), nu.double(), force_no_cam_grad=not cam_grad)
    gref = torch.autograd.grad((ref['rgb'] * wr.double()).sum() + (ref['mask'] * wm.double()).sum(),
                               [sc[n] for n in names] + [cm[n] for n in cam_names],
                               allow_unused=True)
    sc2, cm2 = leaves(scene, cams, names, cam_names)
    rgb, _, mask, _ = Hh.run_cuda(sc2, cm2, H, W, S, nt, nu, mlp_mode=mode, cam_grad=cam_grad)
    got = torch.autograd.grad((rgb * wr).sum() + (mask * wm).sum(),
                              [sc2[n] for n in names] + [cm2[n] for n in cam_names],
                              allow_unused=True)
    if not cam_grad:
        assert all(g is None for g in got[len(names):]), 'camera gradients must be cut'
        # (the oracle's force_no_cam_grad still sends a fine-pass gradient to the camera
        # position, test_fullsize_gpu.py::test_force_no_cam_grad_on_cuda: fields only)
        names, got, gref = names, got[:len(names)], gref[:len(names)]
        cam_names = []
    errs = {n: Hh.rel_l2(a.double(), b) for n, a, b in zip(names + cam_names, got, gref)}
    print('  rel-L2 vs float64: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    for n, e in errs.items():
        assert e < (5e-3 if n == 'beta' else 1e-3), (n, e)


# The three routes of nfi_render_backward with decoder gradients:
#   generator step: render_wgrad_pipe<PLANES=true>, the whole backward in one sweep;
#   decoder + pose: render_backward_pipe (planes, cameras) beside render_wgrad_pipe<false>;
#   decoder only:   render_wgrad_pipe<false> alone.
WGRAD_ROUTES = {
    'generator_step': ('chairs_white_center', 15, ['planes', 'w1', 'b1', 'w2', 'b2', 'palette',
                                                   'beta', 'alpha'], False),
    'decoder_and_pose': ('p3d_bbox', 10, ['planes', 'w1', 'b1', 'w2', 'b2'], True),
    'decoder_only': ('cub_ortho', 0, ['w1', 'b1', 'w2', 'b2'], False),
}


# Steps per tile are S (coarse only) or 2S, and the chains are cut every kWgFlush = 16 steps of
# the CTA's whole run: S = 4 coarse-only has no intermediate flush but chains across tiles, 8
# flushes exactly at every tile boundary, 12 (24 steps) inside tiles, 20 (40 steps) both.
@pytest.mark.parametrize('S,fine', [(4, False), (8, True), (12, True), (20, True)],
                         ids=['S4-coarse', 'S8', 'S12', 'S20'])
@pytest.mark.parametrize('route', list(WGRAD_ROUTES))
def test_decoder_weight_gradients_against_float64(sms, route, S, fine):
    case, A, names, pose = WGRAD_ROUTES[route]
    B = ragged_batch(sms)
    n_tiles = tiles(B, H, W)
    steps = (2 if fine else 1) * S
    lo, hi = per_cta(n_tiles, sms)
    assert_multiwave(n_tiles, sms, 'wgrad %s S=%d fine=%s: %d steps per tile, %d..%d per CTA'
                     % (route, S, fine, steps, steps * lo, steps * hi))
    scene, cams = Hh.make_case(case, seed=13, batch=B, plane_res=64, attention_values=A,
                               device='cuda')
    nt, nu = synthetic.make_noise(83, B, H, W, S, fine=fine, device='cuda')
    cam_names = [k for k in ('c2w', 'focal', 'bbox', 'center') if pose and cams[k] is not None]
    wr, wm = upstream(B, H, W, seed=1)
    sc, cm = leaves(dbl(scene), dbl(cams), names, cam_names)
    ref = Hh.run_oracle(sc, cm, H, W, S, nt.double(), nu.double() if fine else None,
                        fine_sampling=fine)
    gref = torch.autograd.grad((ref['rgb'] * wr.double()).sum() + (ref['mask'] * wm.double()).sum(),
                               [sc[n] for n in names] + [cm[n] for n in cam_names])
    sc2, cm2 = leaves(scene, cams, names, cam_names)
    rgb, _, mask, _ = Hh.run_cuda(sc2, cm2, H, W, S, nt, nu, mlp_mode=4, fine_sampling=fine)
    got = torch.autograd.grad((rgb * wr).sum() + (mask * wm).sum(),
                              [sc2[n] for n in names] + [cm2[n] for n in cam_names])
    errs = {n: Hh.rel_l2(a.double(), b) for n, a, b in zip(names + cam_names, got, gref)}
    print('  rel-L2 vs float64: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    for n, e in errs.items():
        assert e < (5e-3 if n == 'beta' else 1e-3), (n, e)


# ================================================================ 2. the benchmark's workloads

BH = BW = 128
BS = 64


def bench_scene(dataset, B):
    """The inputs bench.py's Bench.scene builds: seed 1234, 256^2 planes channel-last, 10 palette
    entries, the dataset's cameras (no bbox, no center), 128x128 rays, 64 + 64 samples.  Also
    returns the channel-first planes for the oracle."""
    from nerf_from_image_b200.fused import RenderConfig
    ds = synthetic.DATASET_CONFIGS[dataset]
    sc = synthetic.make_scene(1234, B, plane_res=256, attention_values=10,
                              scene_range=ds['scene_range'], white_background=ds['white_background'],
                              object_radius=ds['object_radius'], device='cuda')
    planes_cf = sc['planes']
    sc['planes'] = planes_cf.permute(0, 1, 3, 4, 2).contiguous()
    cams = synthetic.make_cameras(1234, B, ortho=ds['ortho'], radius=ds['radius'], device='cuda')
    nt, nu = synthetic.make_noise(1234, B, BH, BW, BS, device='cuda')
    cfg = RenderConfig(scene_range=sc['scene_range'], white_background=sc['white_background'],
                       attention_values=10, mlp_mode=0)
    return sc, planes_cf, cams, nt, nu, cfg


def bench_render(sc, cams, cfg, h, nt, nu, rows=None):
    from nerf_from_image_b200.fused import fused_render
    return fused_render(sc['planes'], sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                        sc['beta'], sc['alpha'], cams['c2w'], cams['focal'], None, None, cfg, h,
                        BW, BS, nt, nu, planes_layout='channel_last', rows=rows)


def bench_image64(sc, planes_cf, cams, b):
    """Image b's scene (channel-first planes) and camera in float64."""
    s = {k: (v[b:b + 1] if k == 'palette' else v) for k, v in sc.items() if k != 'planes'}
    s['planes'] = planes_cf[b:b + 1]
    return dbl(s), dbl({k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cams.items()})


def bench_oracle(s, c, nt, nu, b):
    """Image b through the oracle (in the precision of ``s`` / ``c``, image b's scene and
    camera)."""
    return O.render_oracle(s['planes'], s['w1'], s['b1'], s['w2'], s['b2'], s['palette'],
                           s['beta'], s['alpha'], c['c2w'], c['focal'], None, None,
                           BH, BW, BS, nt[b:b + 1].double(),
                           nu.view(-1, BH * BW, BS)[b].double(), scene_range=s['scene_range'],
                           white_background=s['white_background'])


def spread(B, n):
    """n image indices spread over the batch, the first and the last included."""
    return sorted({round(i * (B - 1) / (n - 1)) for i in range(n)})


def test_bench_config2_forward(sms):
    """p3d_car, 32 images: the batch equals each image rendered alone; 6 images against the
    float64 oracle."""
    B = 32
    assert_multiwave(tiles(B, BH, BW), sms, 'config 2 forward, %d images' % B)
    sc, planes_cf, cams, nt, nu, cfg = bench_scene('p3d_car', B)
    with torch.no_grad():
        full = bench_render(sc, cams, cfg, BH, nt, nu)[:3]

        def alone(s, c, h, nt_, nu_, rows):
            return bench_render(s, c, cfg, h, nt_, nu_, rows)[:3]
        for b in range(B):
            part = render_alone(alone, sc, cams, nt, nu, b, BH, BW, sms)
            for n, x, y in zip(('rgb', 'depth', 'mask'), part, full):
                assert torch.equal(x[0], y[b]), (b, n, (x[0] - y[b]).abs().max().item())
        for b in spread(B, 6):
            ref = bench_oracle(*bench_image64(sc, planes_cf, cams, b), nt, nu, b)
            errs = [Hh.rel_l2(full[0][b].double(), ref['rgb'][0]),
                    Hh.rel_l2(full[1][b].double(), ref['depth'][0]),
                    Hh.rel_l2(full[2][b].double(), ref['mask'][0])]
            print('  image %2d rel-L2 vs float64: rgb %.2e depth %.2e mask %.2e' % ((b,) + tuple(errs)))
            assert max(errs) < TOL, (b, errs)
            del ref


def _bench_step(dataset, B, names, cam_names, sms, what):
    """The benchmark's step (loss = mean(rgb^2) + mean(mask)) on the batch, and on each image
    alone with the same upstream gradient.  -> (scene, channel-first planes, cameras, noise,
    config, batch gradients, per-image gradients)."""
    assert_multiwave(tiles(B, BH, BW), sms, what)
    sc, planes_cf, cams, nt, nu, cfg = bench_scene(dataset, B)
    n_rgb, n_mask = B * BH * BW * 3, B * BH * BW
    s1, c1 = leaves(sc, cams, names, cam_names)
    rgb, _, mask, _ = bench_render(s1, c1, cfg, BH, nt, nu)
    got = torch.autograd.grad(rgb.square().sum() / n_rgb + mask.sum() / n_mask,
                              [s1[n] for n in names] + [c1[n] for n in cam_names])
    got = dict(zip(names + cam_names, got))
    del rgb, mask, s1, c1
    alone = []
    for b in range(B):
        s_b, c_b, nt_b, nu_b, _ = image(sc, cams, nt, nu, b, BH, BW)
        s_b, c_b = leaves(s_b, c_b, names, cam_names)
        losses = []

        def render(s, c, h, nt_, nu_, rows):
            r, _, m, _ = bench_render(s, c, cfg, h, nt_, nu_, rows)
            losses.append(r.square().sum() / n_rgb + m.sum() / n_mask)
            return (r.detach(),)
        render_alone(render, s_b, c_b, nt_b, nu_b, 0, BH, BW, sms)
        g = torch.autograd.grad(sum(losses), [s_b[n] for n in names] + [c_b[n] for n in cam_names])
        alone.append(dict(zip(names + cam_names, g)))
    return sc, planes_cf, cams, nt, nu, cfg, got, alone


def _oracle_grads(sc, planes_cf, cams, nt, nu, b, B, names, cam_names):
    """float64 oracle autograd of image b under the benchmark's loss (normalised by the batch)."""
    d, c = leaves(*bench_image64(sc, planes_cf, cams, b), names, cam_names)
    ref = bench_oracle(d, c, nt, nu, b)
    loss = ref['rgb'].square().sum() / (B * BH * BW * 3) + ref['mask'].sum() / (B * BH * BW)
    g = torch.autograd.grad(loss, [d[n] for n in names] + [c[n] for n in cam_names])
    out = dict(zip(names + cam_names, g))
    out['planes'] = out['planes'].permute(0, 1, 3, 4, 2)   # channel-last, as the kernel's
    return out


def test_bench_config3_inversion_step(sms):
    """cub, 16 images, gradients to planes, palette and pose (+ beta / alpha): each image's
    gradients equal those of the image rendered alone up to the order of the plane-gradient
    atomics; beta / alpha equal the sum over the images; 4 images against float64 autograd."""
    B = 16
    names, cam_names = ['planes', 'palette', 'beta', 'alpha'], ['c2w']
    sc, planes_cf, cams, nt, nu, cfg, got, alone = _bench_step(
        'cub', B, names, cam_names, sms, 'config 3 inversion step, %d images' % B)
    worst = {}
    for b in range(B):
        for n in ('planes', 'palette', 'c2w'):
            e = Hh.rel_l2(got[n][b], alone[b][n][0])
            worst[n] = max(worst.get(n, 0.0), e)
            assert e < 1e-5, (b, n, e)
    for n in ('beta', 'alpha'):
        worst[n] = Hh.rel_l2(got[n], sum(a[n] for a in alone))
    print('  batch vs alone rel-L2 (worst image): ' + ', '.join('%s %.2e' % kv for kv in worst.items()))
    assert worst['beta'] < 1e-4 and worst['alpha'] < 1e-4, worst
    for b in spread(B, 4):
        ref = _oracle_grads(sc, planes_cf, cams, nt, nu, b, B, ['planes', 'palette'], cam_names)
        errs = {n: Hh.rel_l2(got[n][b:b + 1].double(), ref[n]) for n in ('planes', 'palette', 'c2w')}
        print('  image %2d rel-L2 vs float64: ' % b + ', '.join('%s %.2e' % kv for kv in errs.items()))
        for n, e in errs.items():
            assert e < 1e-3, (b, n, e)
        del ref


def test_bench_config4_generator_step(sms):
    """shapenet_chairs, generator step (decoder, beta, alpha, planes, palette; cameras are
    data), 6 images = 768 tiles: the gradients shared by the batch against the sum of float64
    oracle autograd over the images, the per-image ones image by image."""
    B = 6
    names = ['planes', 'palette', 'w1', 'b1', 'w2', 'b2', 'beta', 'alpha']
    assert_multiwave(tiles(B, BH, BW), sms, 'config 4 generator step, %d images' % B)
    sc, planes_cf, cams, nt, nu, cfg = bench_scene('shapenet_chairs', B)
    s1, c1 = leaves(sc, cams, names, [])
    rgb, _, mask, _ = bench_render(s1, c1, cfg, BH, nt, nu)
    got = torch.autograd.grad(rgb.square().mean() + mask.mean(), [s1[n] for n in names])
    got = dict(zip(names, got))
    del rgb, mask
    shared = ['w1', 'b1', 'w2', 'b2', 'beta', 'alpha']
    total = None
    for b in range(B):
        ref = _oracle_grads(sc, planes_cf, cams, nt, nu, b, B, names, [])
        errs = {n: Hh.rel_l2(got[n][b:b + 1].double(), ref[n]) for n in ('planes', 'palette')}
        print('  image %d rel-L2 vs float64: ' % b + ', '.join('%s %.2e' % kv for kv in errs.items()))
        for n, e in errs.items():
            assert e < 1e-3, (b, n, e)
        total = {n: ref[n] for n in shared} if total is None else \
            {n: total[n] + ref[n] for n in shared}
        del ref
    errs = {n: Hh.rel_l2(got[n].double(), total[n]) for n in shared}
    print('  shared gradients rel-L2 vs float64 sum: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    for n, e in errs.items():
        assert e < 1e-3, (n, e)


# ================================================================ 3. synthesis conv_tc_kernel

def conv_tiles(B, R, N):
    """conv_tc_kernel tiles of a stride-1 GEMM: 16 x 16 positions by BN output channels."""
    bn = 128 if N % 128 == 0 else N
    return B * math.ceil(R / 16) ** 2 * (N // bn)


# (channels, batch).  Narrow channels keep the reduction length K = 9 x Cin small.  The first net's
# conv1 at 256^2 runs 768 tiles and the FIR-adjoint phase GEMM at 128^2 192; the second has BN =
# 128 and BN = 64 layers.
SYNTH_CASES = [((64, 64, 64, 32, 32, 32, 32), 3), ((128, 128, 128, 64, 64, 64), 4)]
SYNTH_TOL = 5e-5   # measured on an H100: 9.3e-6 and 1.3e-5
# ws.grad bar (every ws row under it too) against float64 on the kernel's own leaky-ReLU branches
# where float64's u is within TAU of zero, plain float64 elsewhere (tests/synthesis_branch_oracle
# .py).  Measured on an H100: 1.24e-5 (rows <= 1.9e-5, 44 positions borrowed, |u64| <= 2.3e-5) and
# 1.68e-5 (rows <= 2.2e-5, 33 borrowed); against plain float64 4.6e-3 and 3.7e-3, each row up to
# the last flipped layer's off by 0.6e-3 .. 1e-2.
SYNTH_GRAD_BAR = {(64, 64, 64, 32, 32, 32, 32): 3.5e-5, (128, 128, 128, 64, 64, 64): 5e-5}


def _synth_case(sms, channels, batch):
    res = 4 << (len(channels) - 1)
    n = conv_tiles(batch, res, channels[-1])
    lo, hi = per_cta(n, sms)
    print('\nsynthesis %r B=%d: conv1 at %d^2 %d tiles on %d SMs, %d..%d tiles per CTA'
          % (channels, batch, res, n, sms, lo, hi))
    assert n > sms, (n, sms)
    p = synthetic.make_synthesis_params(5, res, channels, 512, 'cuda')
    g = torch.Generator().manual_seed(8)
    ws = torch.randn(batch, 2 * len(channels), 512, generator=g).cuda()
    return res, p, ws, g


@pytest.mark.parametrize('channels,batch', SYNTH_CASES)
def test_synthesis_forward_against_float64(sms, channels, batch):
    from nerf_from_image_b200.synthesis import FusedSynthesis, planes_channel_first
    res, p, ws, _ = _synth_case(sms, channels, batch)
    fs = FusedSynthesis.from_params(p)
    with torch.no_grad():
        got = fs(ws, noise_mode='const')
        want = SO.synthesis_forward(dbl(p), ws.double(),
                                    {k: v.double() for k, v in HS.const_noises(p).items()})
    saved = fs.forward_differentiable(ws.clone().requires_grad_(), noise_mode='const')
    assert torch.equal(saved.detach(), got)
    err = Hh.rel_l2(planes_channel_first(got).double(), want)
    print('  planes rel-L2 vs float64 %.2e' % err)
    assert err < SYNTH_TOL, err


def _synth_ws_grad(p, ws, g_planes):
    from nerf_from_image_b200.synthesis import FusedSynthesis
    w = ws.clone().requires_grad_()
    FusedSynthesis.from_params(p).forward_differentiable(w, noise_mode='const').backward(g_planes)
    return w.grad


@pytest.mark.parametrize('channels,batch', SYNTH_CASES)
def test_synthesis_ws_grad_batch_equals_each_image_alone(sms, channels, batch):
    """Each image's ws.grad in the multi-wave batch against the image's own run (ws rows are per
    image; only the order of the per-(image, channel) atomic sums differs): measured on an H100,
    6.4e-8 and 7.9e-8."""
    res, p, ws, g = _synth_case(sms, channels, batch)
    g_planes = torch.randn(batch, 3, res, res, 32, generator=g).cuda()
    got = _synth_ws_grad(p, ws, g_planes)
    alone = torch.cat([_synth_ws_grad(p, ws[b:b + 1], g_planes[b:b + 1]) for b in range(batch)])
    err = Hh.rel_l2(got, alone)
    print('  ws.grad batch vs each image alone rel-L2 %.2e' % err)
    assert err < 1e-6, err


@pytest.mark.parametrize('channels,batch', SYNTH_CASES)
def test_synthesis_ws_grad_against_float64(sms, channels, batch):
    from nerf_from_image_b200.synthesis import FusedSynthesis, planes_channel_first, saved_preactivations
    res, p, ws, g = _synth_case(sms, channels, batch)
    g_planes = torch.randn(batch, 3, res, res, 32, generator=g).cuda()
    w = ws.clone().requires_grad_()
    planes = FusedSynthesis.from_params(p).forward_differentiable(w, noise_mode='const')
    u_kernel = saved_preactivations(planes)
    planes.backward(g_planes)
    got = w.grad.double()
    pd, wd, nz, masks, _ = BO.kernel_branches(p, u_kernel, ws, HS.const_noises(p))
    g_img = planes_channel_first(g_planes.double())
    want = BO.ws_grad(pd, wd, nz, g_img)
    want_br = BO.ws_grad(pd, wd, nz, g_img, masks)
    err, err_br = Hh.rel_l2(got, want), Hh.rel_l2(got, want_br)
    row, row_br = BO.row_errors(got, want), BO.row_errors(got, want_br)
    print('  ws.grad rel-L2 on the kernel\'s branches %.2e, per row %s' % (
        err_br, ' '.join('%.1e' % r for r in row_br)))
    print('  ws.grad rel-L2 vs plain float64 %.2e, per row %s' % (err, ' '.join('%.1e' % r for r in row)))
    assert err_br < SYNTH_GRAD_BAR[channels], err_br
    assert max(row_br) < SYNTH_GRAD_BAR[channels], row_br
