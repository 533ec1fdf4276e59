"""CUDA path (through the C ABI) vs the CPU oracle -- the parity tests proper.

Bar (BASELINE.json north_star): <= 1e-3 relative L2 on rgb against the fp32
reference render with identical injected noise.  The asserts below use a
tighter 2e-4 (3xTF32 / fp32 arithmetic leaves ~1e-6) so regressions show.
"""
import pytest
import torch

from tests import helpers as Hh
from fixtures import synthetic

pytestmark = pytest.mark.gpu
TOL = 2e-4


@pytest.fixture(autouse=True, params=[1, 2, 4], ids=['simt', 'tc', 'pipe'])
def mlp_mode(request):
    """Every test below runs with the fp32 SIMT MLP, with NFI_MLP_TC_3XTF32 (an alias of the
    pipelined kernels) and with the pipelined wgmma 3xTF32 MLP, NFI_MLP_TC_PIPE (S = 16 keeps
    every render inside the tensor-core envelope S <= 128, S % 4 == 0; renders outside it fall
    back under NFI_MLP_AUTO)."""
    Hh.MLP_MODE = request.param
    yield request.param
    Hh.MLP_MODE = 0


def _noise(seed, B, H, W, S, fine=True):
    return synthetic.make_noise(seed, B, H, W, S, fine=fine)


@pytest.mark.parametrize('case', list(Hh.CASES))
@pytest.mark.parametrize('randomize', [True, False])
def test_forward_matches_oracle(cuda_lib, case, randomize):
    B, H, W, S = 2, 12, 20, 16   # deliberately not a multiple of the 16x8 CTA tile
    scene, cams = Hh.make_case(case, batch=B)
    nt, nu = _noise(3, B, H, W, S) if randomize else (None, None)
    ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu)
    rgb, depth, mask, _ = Hh.run_cuda(scene, cams, H, W, S, nt, nu)
    # randomize=False puts coarse sample 0 exactly ON the cube face, where the
    # out-of-cube test |x| > 1 is decided by one ulp of the near-plane
    # arithmetic (SURVEY.md section 7, hard part 4): those runs are held to the
    # stated 1e-3 bar, jittered runs to the tight one.
    tol = TOL if randomize else 1e-3
    assert Hh.rel_l2(rgb.cpu(), ref['rgb']) < tol
    assert Hh.rel_l2(mask.cpu(), ref['mask']) < tol
    assert Hh.rel_l2(depth.cpu(), ref['depth']) < tol


@pytest.mark.parametrize('fine', [True, False])
@pytest.mark.parametrize('A,use_sdf', [(10, True), (0, True), (10, False), (15, True), (3, True)])
def test_forward_variants(cuda_lib, fine, A, use_sdf):
    B, H, W, S = 2, 16, 16, 16
    scene, cams = Hh.make_case('p3d_bbox', batch=B, attention_values=A)
    nt, nu = _noise(5, B, H, W, S, fine=fine)
    ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu, use_sdf=use_sdf, fine_sampling=fine)
    rgb, depth, mask, _ = Hh.run_cuda(scene, cams, H, W, S, nt, nu, use_sdf=use_sdf,
                                      fine_sampling=fine)
    assert Hh.rel_l2(rgb.cpu(), ref['rgb']) < TOL
    assert Hh.rel_l2(mask.cpu(), ref['mask']) < TOL
    assert Hh.rel_l2(depth.cpu(), ref['depth']) < TOL


@pytest.mark.parametrize('S', [32, 64, 128])
def test_forward_and_backward_sample_counts(cuda_lib, S):
    """BASELINE config 5 sweeps 32 -> 128 samples per ray: the pipelined kernels take
    S <= 128 (2 or 4 resampling slots per lane)."""
    B, H, W = 1, 16, 24
    scene, cams = Hh.make_case('p3d_bbox', batch=B)
    nt, nu = _noise(37, B, H, W, S)
    outs = []
    for dev in ('cpu', 'cuda'):
        sc, cm = Hh.to_device(scene, dev), Hh.to_device(cams, dev)
        sc['planes'] = sc['planes'].clone().requires_grad_()
        if dev == 'cpu':
            r = Hh.run_oracle(sc, cm, H, W, S, nt, nu)
            rgb, mask, depth = r['rgb'], r['mask'], r['depth']
        else:
            rgb, depth, mask, _ = Hh.run_cuda(sc, cm, H, W, S, nt, nu)
        outs.append((rgb.detach().cpu(), mask.detach().cpu(), depth.detach().cpu(),
                     _grads((rgb, mask), [sc['planes']])[0].cpu()))
    for a, b, tol in zip(outs[1], outs[0], (TOL, TOL, TOL, 2e-3)):
        assert Hh.rel_l2(a, b) < tol


@pytest.mark.parametrize('mode', ['coords', 'semantics'])
def test_extra_outputs(cuda_lib, mode):
    B, H, W, S = 2, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt, nu = _noise(7, B, H, W, S)
    ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu, compute_coords=(mode == 'coords'),
                        compute_semantics=(mode == 'semantics'))
    rgb, depth, mask, extra = Hh.run_cuda(scene, cams, H, W, S, nt, nu,
                                          extra_mode=1 if mode == 'coords' else 2)
    assert Hh.rel_l2(rgb.cpu(), ref['rgb']) < TOL
    assert Hh.rel_l2(extra.cpu(), ref['semantics']) < TOL


@pytest.mark.parametrize('case,fine,semantics', [('p3d_plain', True, True), ('p3d_bbox', False, False),
                                                 ('chairs_white_center', True, False)])
def test_normals_match_oracle(cuda_lib, case, fine, semantics, mlp_mode):
    """compute_normals (evaluation / visualisation calls of run.py:1263,1453,2043,2132):
    normalised analytic SDF gradient, composited with the weights; together with
    compute_semantics as the reference's evaluation loops request them."""
    B, H, W, S = 2, 16, 16, 16
    scene, cams = Hh.make_case(case, batch=B)
    nt, nu = _noise(41, B, H, W, S, fine=fine)
    ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu, fine_sampling=fine, compute_normals=True,
                        compute_semantics=semantics)
    # explicit tensor-core modes refuse normals / semantics; NFI_MLP_AUTO (0) falls back by itself
    rgb, depth, mask, extra, normals = Hh.run_cuda(scene, cams, H, W, S, nt, nu, fine_sampling=fine,
                                                   extra_mode=2 if semantics else 0,
                                                   compute_normals=True,
                                                   mlp_mode=1 if mlp_mode == 1 else 0)
    assert Hh.rel_l2(rgb.cpu(), ref['rgb'].detach()) < TOL
    assert Hh.rel_l2(normals.cpu(), ref['normals'].detach()) < 1e-3
    if semantics:
        assert Hh.rel_l2(extra.cpu(), ref['semantics'].detach()) < TOL


def test_fine_depths_match(cuda_lib):
    """The importance-resampled depths themselves (sorted) on rays that hit."""
    B, H, W, S = 1, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt, nu = _noise(11, B, H, W, S)
    ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu)
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200.fused import FusedTriplaneRender, RenderConfig
    sc, cm = Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda')
    planes = sc['planes'].clone().requires_grad_()
    cfg = RenderConfig(scene_range=sc['scene_range'])
    out = FusedTriplaneRender.apply(planes, sc['w1'], sc['b1'], sc['w2'], sc['b2'],
                                    sc['palette'], sc['beta'], sc['alpha'], cm['c2w'],
                                    cm['focal'], None, None, cfg, H, W, S, nt.cuda(), nu.cuda(),
                                    0, True)
    fn = out[0].grad_fn
    zf = dict(zip(fn.saved_names, fn.saved_tensors))['z_fine'].view(B, H, W, S).cpu()
    zr = ref['z_fine'].sort(dim=-1).values
    from oracle import render_oracle as O
    o, d = O.ray_bundle(H, W, cams['focal'], cams['c2w'], None, None)
    hit = O.near_far_planes(o, torch.nn.functional.normalize(d, dim=-1), scene['scene_range'])[2]
    assert hit.any()
    assert (zf[hit] - zr[hit]).abs().max() < 2e-5


def _grads(outs, inputs, seed=0):
    rgb, mask = outs
    g = torch.Generator().manual_seed(seed)
    wr = torch.randn(rgb.shape, generator=g).to(rgb.device)
    wm = torch.randn(mask.shape, generator=g).to(rgb.device)
    loss = (rgb * wr).sum() + (mask * wm).sum()
    return torch.autograd.grad(loss, inputs, allow_unused=True)


@pytest.mark.parametrize('case', ['p3d_bbox', 'cub_ortho', 'chairs_white_center'])
def test_backward_matches_oracle_autograd(cuda_lib, case):
    B, H, W, S = 2, 12, 20, 16
    scene, cams = Hh.make_case(case, batch=B)
    nt, nu = _noise(13, B, H, W, S)
    names = ['planes', 'w1', 'b1', 'w2', 'b2', 'palette', 'beta', 'alpha']
    cam_names = ['c2w'] + (['focal'] if cams['focal'] is not None else []) + \
        (['bbox'] if cams['bbox'] is not None else []) + \
        (['center'] if cams['center'] is not None else [])

    def leaves(dev):
        sc = {k: (v.detach().clone().to(dev).requires_grad_() if k in names else v)
              for k, v in scene.items()}
        cm = {k: (v.detach().clone().to(dev).requires_grad_() if k in cam_names else
                  (v.to(dev) if torch.is_tensor(v) else v)) for k, v in cams.items()}
        return sc, cm

    sc, cm = leaves('cpu')
    ref = Hh.run_oracle(sc, cm, H, W, S, nt, nu)
    gref = _grads((ref['rgb'], ref['mask']), [sc[n] for n in names] + [cm[n] for n in cam_names])
    sc2, cm2 = leaves('cuda')
    rgb, depth, mask, _ = Hh.run_cuda(sc2, cm2, H, W, S, nt, nu)
    gcu = _grads((rgb, mask), [sc2[n] for n in names] + [cm2[n] for n in cam_names])
    for n, a, b in zip(names + cam_names, gcu, gref):
        assert a is not None and b is not None, n
        err = Hh.rel_l2(a.cpu(), b)
        assert err < 2e-3, (n, err)   # (decoder weights: render_wgrad_pipe under the tc modes)


@pytest.mark.parametrize('case', ['p3d_bbox', 'cub_ortho', 'chairs_white_center'])
def test_backward_frozen_decoder_matches_oracle_autograd(cuda_lib, case):
    """The inversion setting (run.py:628-629: decoder frozen): gradients to the planes,
    palette, beta / alpha and cameras only.  Under the tensor-core mlp modes this is
    render_backward_pipe (wgmma, 3xTF32 for all four GEMMs); under 'simt' the fp32 kernel."""
    B, H, W, S = 2, 12, 20, 16
    scene, cams = Hh.make_case(case, batch=B)
    nt, nu = _noise(29, B, H, W, S)
    names = ['planes', 'palette', 'beta', 'alpha']
    cam_names = ['c2w'] + (['focal'] if cams['focal'] is not None else []) + \
        (['bbox'] if cams['bbox'] is not None else []) + \
        (['center'] if cams['center'] is not None else [])

    def leaves(dev):
        sc = {k: (v.detach().clone().to(dev).requires_grad_() if k in names else
                  (v.to(dev) if torch.is_tensor(v) else v)) for k, v in scene.items()}
        cm = {k: (v.detach().clone().to(dev).requires_grad_() if k in cam_names else
                  (v.to(dev) if torch.is_tensor(v) else v)) for k, v in cams.items()}
        return sc, cm

    sc, cm = leaves('cpu')
    ref = Hh.run_oracle(sc, cm, H, W, S, nt, nu)
    gref = _grads((ref['rgb'], ref['mask']), [sc[n] for n in names] + [cm[n] for n in cam_names])
    sc2, cm2 = leaves('cuda')
    rgb, depth, mask, _ = Hh.run_cuda(sc2, cm2, H, W, S, nt, nu)
    gcu = _grads((rgb, mask), [sc2[n] for n in names] + [cm2[n] for n in cam_names])
    for n, a, b in zip(names + cam_names, gcu, gref):
        assert a is not None and b is not None, n
        err = Hh.rel_l2(a.cpu(), b)
        assert err < 2e-3, (n, err)


def test_backward_no_fine_sampling_frozen(cuda_lib):
    """Coarse-only render (args.fine_sampling False) through the frozen-decoder backward."""
    B, H, W, S = 1, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt, _ = _noise(31, B, H, W, S, fine=False)
    outs = []
    for dev in ('cpu', 'cuda'):
        sc = Hh.to_device(scene, dev)
        cm = Hh.to_device(cams, dev)
        sc['planes'] = sc['planes'].clone().requires_grad_()
        if dev == 'cpu':
            r = Hh.run_oracle(sc, cm, H, W, S, nt, None, fine_sampling=False)
            rgb, mask = r['rgb'], r['mask']
        else:
            rgb, _, mask, _ = Hh.run_cuda(sc, cm, H, W, S, nt, None, fine_sampling=False)
        outs.append(_grads((rgb, mask), [sc['planes']])[0])
    assert Hh.rel_l2(outs[1].cpu(), outs[0]) < 2e-3


def test_backward_extras_and_frozen_weights(cuda_lib):
    """compute_coords gradient path + the inversion setting (only planes,
    palette and cameras require grad; decoder frozen)."""
    B, H, W, S = 1, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt, nu = _noise(17, B, H, W, S)
    outs = []
    for dev in ('cpu', 'cuda'):
        sc = Hh.to_device(scene, dev)
        cm = Hh.to_device(cams, dev)
        sc['planes'] = sc['planes'].clone().requires_grad_()
        sc['palette'] = sc['palette'].clone().requires_grad_()
        cm['c2w'] = cm['c2w'].clone().requires_grad_()
        if dev == 'cpu':
            r = Hh.run_oracle(sc, cm, H, W, S, nt, nu, compute_coords=True)
            rgb, ex = r['rgb'], r['semantics']
        else:
            rgb, _, _, ex = Hh.run_cuda(sc, cm, H, W, S, nt, nu, extra_mode=1)
        g = torch.Generator().manual_seed(1)
        loss = (rgb * torch.randn(rgb.shape, generator=g).to(dev)).sum() + \
            (ex * torch.randn(ex.shape, generator=g).to(dev)).sum()
        outs.append(torch.autograd.grad(loss, [sc['planes'], sc['palette'], cm['c2w']]))
    for a, b, n in zip(outs[1], outs[0], ['planes', 'palette', 'c2w']):
        assert Hh.rel_l2(a.cpu(), b) < 2e-3, n


@pytest.mark.parametrize('mlp_mode', [2, 3], ids=['tc', 'warpspec'])  # (instead of the fixture)
@pytest.mark.parametrize('case', ['fine_s128', 'semantics_a10', 'coarse_s160'])
def test_tc_modes_are_aliases_of_pipe(cuda_lib, case, mlp_mode):
    """NFI_MLP_TC_3XTF32 (2) and NFI_MLP_TC_WARPSPEC (3) run the pipelined kernels of
    NFI_MLP_TC_PIPE (4): the same renders run (fine sampling at S = 128, semantics with 10 palette
    entries) with the same outputs bit for bit and the same gradients, and the same renders are
    refused (no fine sampling at S = 160: outside the pipelined kernels, left to NFI_MLP_AUTO)."""
    from nerf_from_image_b200._lib import NfiError
    fine, S, extra_mode = {'fine_s128': (True, 128, 0), 'semantics_a10': (True, 16, 2),
                           'coarse_s160': (False, 160, 0)}[case]
    B, H, W = 1, 16, 24
    scene, cams = Hh.make_case('p3d_bbox', batch=B, attention_values=10)
    nt, nu = _noise(47, B, H, W, S, fine=fine)
    names = ['planes', 'w1', 'b1', 'w2', 'b2']

    def run(mode):
        sc, cm = Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda')
        for n in names:
            sc[n] = sc[n].clone().requires_grad_()
        cm['c2w'] = cm['c2w'].clone().requires_grad_()
        outs = Hh.run_cuda(sc, cm, H, W, S, nt, nu, fine_sampling=fine, extra_mode=extra_mode,
                           mlp_mode=mode)
        rgb, depth, mask, extra = outs  # (extra: None without an extra output)
        grads = _grads((rgb, mask), [sc[n] for n in names] + [cm['c2w']])
        return [o.detach() for o in outs if o is not None], grads

    if case == 'coarse_s160':
        for mode in (mlp_mode, 4):
            with pytest.raises(NfiError, match='NFI_MLP_AUTO'):
                run(mode)
        return
    (outs, grads), (want_outs, want_grads) = run(mlp_mode), run(4)
    for a, b in zip(outs, want_outs):  # rgb, depth, mask, extra
        assert torch.equal(a, b)
    # (the plane and decoder-weight gradients are sums of float atomics, in an order that varies
    # from run to run)
    for n, a, b in zip(names + ['c2w'], grads, want_grads):
        assert Hh.rel_l2(a, b) < 1e-5, n


def test_relayout_roundtrip(cuda_lib):
    from nerf_from_image_b200.fused import planes_to_channel_last, planes_from_channel_last
    x = torch.randn(3, 3, 32, 24, 24, device='cuda')
    cl = planes_to_channel_last(x)
    assert torch.equal(cl, x.permute(0, 1, 3, 4, 2).contiguous())
    assert torch.equal(planes_from_channel_last(cl), x)


def test_batch_sharding_is_exact(cuda_lib):
    """Rendering images one by one equals the batched render bit for bit
    (what multi-GPU sharding by image relies on, SURVEY.md section 8e)."""
    B, H, W, S = 4, 32, 32, 16
    scene, cams = Hh.make_case('p3d_bbox', batch=B)
    nt, nu = _noise(19, B, H, W, S)
    full = Hh.run_cuda(scene, cams, H, W, S, nt, nu)
    for b in range(B):
        sc = {k: (v[b:b + 1] if k in ('planes', 'palette') else v) for k, v in scene.items()}
        cm = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cams.items()}
        part = Hh.run_cuda(sc, cm, H, W, S, nt[b:b + 1],
                           nu.view(B, H * W, S)[b].contiguous())
        for x, y in zip(part[:3], full[:3]):
            assert torch.equal(x[0], y[b])


def test_full_size_against_gpu_oracle(cuda_lib):
    """BASELINE config-2 geometry (128x128, 64+64 samples, 256^2 planes) for
    one image: the oracle itself runs on the GPU here (fp32, TF32 off)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, H, W, S = 1, 128, 128, 64
    scene, cams = Hh.make_case('p3d_plain', batch=B, plane_res=256, device='cuda')
    nt, nu = synthetic.make_noise(23, B, H, W, S, device='cuda')
    with torch.no_grad():
        ref = Hh.run_oracle(scene, cams, H, W, S, nt, nu)
        rgb, depth, mask, _ = Hh.run_cuda(scene, cams, H, W, S, nt, nu)
    assert 0.2 < ref['mask'].mean().item() < 0.95
    assert Hh.rel_l2(rgb, ref['rgb']) < TOL
    assert Hh.rel_l2(mask, ref['mask']) < TOL
    assert mask.min().item() >= -1e-6 and mask.max().item() <= 1 + 1e-5


def test_fill_uniform_and_host_entry_philox(cuda_lib):
    """nfi_fill_uniform: range, determinism, independence of how the buffer is split; and the
    host entry point with NFI_NOISE_PHILOX equals the device path fed with the same noise."""
    import ctypes
    from nerf_from_image_b200 import _lib
    lib = cuda_lib
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n = 4 * 12345 + 2
    a = torch.empty(n, device='cuda')
    b = torch.empty(n, device='cuda')
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(a.data_ptr()), n, 77, 0, 0, st))
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(b.data_ptr()), 4000, 77, 0, 0, st))
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(b.data_ptr() + 16000), n - 4000, 77, 0, 4000, st))
    assert torch.equal(a, b)
    assert 0.0 <= a.min().item() and a.max().item() < 1.0
    assert abs(a.mean().item() - 0.5) < 0.01 and abs(a.var().item() - 1 / 12) < 0.005
    c = torch.empty(n, device='cuda')
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(c.data_ptr()), n, 77, 1, 0, st))
    assert not torch.equal(a, c)

    B, H, W, S = 2, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt = torch.empty(B, H, W, S, device='cuda')
    nu = torch.empty(B * H * W, S, device='cuda')
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(nt.data_ptr()), nt.numel(), 5, 0, 0, st))
    _lib.check(lib.nfi_fill_uniform(ctypes.c_void_p(nu.data_ptr()), nu.numel(), 5, 1, 0, st))
    rgb, depth, mask, _ = Hh.run_cuda(scene, cams, H, W, S, nt, nu)
    host = {k: scene[k].contiguous() for k in ('planes', 'w1', 'b1', 'w2', 'b2', 'palette', 'beta', 'alpha')}
    host['c2w'], host['focal'] = cams['c2w'].contiguous(), cams['focal'].contiguous()
    host['rgb'], host['depth'], host['mask'] = torch.empty(B, H, W, 3), torch.empty(B, H, W), torch.empty(B, H, W)
    p = _lib.RenderParams()
    p.batch, p.height, p.width, p.num_samples = B, H, W, S
    p.plane_res, p.n_attention = scene['planes'].shape[-1], scene['palette'].shape[1]
    p.scene_range, p.white_background = scene['scene_range'], int(scene['white_background'])
    p.use_sdf, p.fine_sampling, p.noise_mode, p.noise_seed = 1, 1, _lib.NOISE_PHILOX, 5
    p.mlp_mode = Hh.MLP_MODE
    for k, v in host.items():
        setattr(p, k, ctypes.c_void_p(v.data_ptr()))
    _lib.check(lib.nfi_render_forward_host(ctypes.byref(p), 0))
    assert torch.equal(host['rgb'], rgb.cpu())
    assert torch.equal(host['mask'], mask.cpu())


def test_half_precision_inputs_are_widened(cuda_lib):
    """bf16 planes (autocast around the synthesis network) render like their fp32 widening,
    and the gradient comes back in bf16."""
    B, H, W, S = 1, 16, 16, 16
    scene, cams = Hh.make_case('p3d_plain', batch=B)
    nt, nu = _noise(43, B, H, W, S)
    sc = Hh.to_device(scene, 'cuda')
    pl16 = sc['planes'].to(torch.bfloat16).requires_grad_()
    sc16 = dict(sc, planes=pl16)
    sc32 = dict(sc, planes=pl16.detach().float())
    a = Hh.run_cuda(sc16, cams, H, W, S, nt, nu)
    b = Hh.run_cuda(sc32, cams, H, W, S, nt, nu)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    a[0].square().sum().backward()
    assert pl16.grad is not None and pl16.grad.dtype == torch.bfloat16 and pl16.grad.abs().sum() > 0


@pytest.mark.gpu
def test_caller_owned_outputs(cuda_lib):
    """fused_render(out=...) writes into slices of a larger buffer (the in-place all-gather of
    parallel.render_sharded) and returns exactly what the allocating call returns."""
    from nerf_from_image_b200 import parallel
    from nerf_from_image_b200.fused import RenderConfig, fused_render
    from nerf_from_image_b200._lib import NfiError
    scene, cams = Hh.make_case('p3d_bbox', seed=4, batch=2, plane_res=32, device='cuda')
    H, W, S = 16, 24, 16
    nt, nu = synthetic.make_noise(4, 2, H, W, S, device='cuda')
    cfg = RenderConfig(scene_range=scene['scene_range'], white_background=scene['white_background'],
                       attention_values=10)
    args = (scene['planes'], scene['w1'], scene['b1'], scene['w2'], scene['b2'], scene['palette'],
            scene['beta'], scene['alpha'], cams['c2w'], cams['focal'], cams['center'],
            cams['bbox'], cfg, H, W, S, nt, nu)
    with torch.no_grad():
        ref = fused_render(*args)
        full = parallel.gathered_buffers(6, H, W, 'cuda')
        for t in full:
            t.fill_(-7.0)
        out = parallel.shard_views(full, 6, 3, 1)  # rank 1 of 3: images 2..3
        got = fused_render(*args, out=out)
    for a, b, o in zip(got[:3], ref[:3], out):
        assert a.data_ptr() == o.data_ptr()
        assert torch.equal(a, b)
    for t in full:  # neighbours' slices untouched
        assert (t[:2] == -7.0).all() and (t[4:] == -7.0).all()
    with pytest.raises(NfiError):
        fused_render(*args, out=(full[0][:2, :, :, :2], full[1][:2], full[2][:2]))


def test_row_tiles_are_exact(cuda_lib):
    """Rows [r0, r1) of an image rendered on their own (nfi_render_params.row_offset /
    full_height: one image split over several GPUs, parallel.render_row_sharded) are bit-identical
    to the same rows of the whole image, forward and plane gradient."""
    from nerf_from_image_b200 import parallel as PAR
    from nerf_from_image_b200.fused import RenderConfig, fused_render
    B, H, W, S = 2, 40, 24, 16
    scene, cams = Hh.make_case('p3d_bbox', batch=B)
    nt, nu = _noise(17, B, H, W, S)
    sc, cm = Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda')
    nt, nu = nt.cuda(), nu.cuda()
    cfg = RenderConfig(scene_range=sc['scene_range'], mlp_mode=Hh.MLP_MODE)

    def render(planes, h, nt_, nu_, rows):
        return fused_render(planes, sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                            sc['beta'], sc['alpha'], cm['c2w'], cm['focal'], cm['center'],
                            cm['bbox'], cfg, h, W, S, nt_, nu_, rows=rows)

    p_full = sc['planes'].clone().requires_grad_()
    full = render(p_full, H, nt, nu, None)
    g = torch.Generator().manual_seed(3)
    wr = torch.randn(B, H, W, 3, generator=g).cuda()
    (full[0] * wr).sum().backward()
    p_rows = sc['planes'].clone().requires_grad_()
    pieces = []
    for rank in range(3):
        r0, r1 = PAR.row_range(H, 3, rank)
        nt_, nu_ = PAR.slice_rows(nt, nu, B, H, W, r0, r1)
        out = render(p_rows, r1 - r0, nt_, nu_, (r0, H))
        (out[0] * wr[:, r0:r1]).sum().backward()
        pieces.append(out)
    assert [PAR.row_range(H, 3, r) for r in range(3)] == [(0, 16), (16, 32), (32, 40)]
    for i in range(3):
        assert torch.equal(torch.cat([p[i] for p in pieces], dim=1), full[i])
    # (atomics: the plane gradient is summed in a different order)
    assert Hh.rel_l2(p_rows.grad, p_full.grad) < 1e-5
