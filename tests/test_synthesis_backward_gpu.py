"""The synthesis backward to the latents on sm_90a (nfi_synthesis_forward_saved +
nfi_synthesis_backward through ``FusedSynthesis.forward_differentiable``):

1. the saved forward emits exactly the plain forward's planes;
2. ws.grad against float64 autograd through the oracle on seeded ragged networks, overall and per
   ws row;
3. where the reference is installed, the full 512-channel 256^2 SynthesisNetwork against the
   module's own float64 autograd;
4. ``render()`` with ``enable_fused_inversion`` on the reference Generator against the reference
   render + module: gradients to ws (both latent forms), the pose and through the palette, RNG
   consumption, and the fall-back for a trainable synthesis network."""
import types

import pytest
import torch

from fixtures import synthetic
from oracle import reference_lift as RL
from oracle import synthesis_oracle as SO
from tests import helpers_synth as HS
from tests import synthesis_branch_oracle as BO

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _cf(planes_cl):
    from nerf_from_image_b200.synthesis import planes_channel_first
    return planes_channel_first(planes_cl)


def _double(p):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v)
            for k, v in p.items()}


def test_saved_forward_equals_the_plain_forward(cuda_lib):
    from nerf_from_image_b200.synthesis import FusedSynthesis
    cases = [HS.load_case(c, 'cuda')[:2] for c in HS.CASES]
    for channels, batch in (((128, 128, 64, 32), 3), ((256, 128, 128, 96, 64), 2)):
        res = 4 << (len(channels) - 1)
        p = synthetic.make_synthesis_params(5, res, channels, 512, 'cuda')
        ws = torch.randn(batch, 2 * len(channels), 512,
                         generator=torch.Generator().manual_seed(6)).cuda()
        cases.append((p, ws))
    for p, ws in cases:
        fs = FusedSynthesis.from_params(p)
        with torch.no_grad():
            plain = fs(ws, noise_mode='const')
        saved = fs.forward_differentiable(ws.clone().requires_grad_(), noise_mode='const')
        assert torch.equal(saved.detach(), plain)


# (channels, batch, plain bar, bar).  ``bar`` holds ws.grad and every ws row against float64 on
# the kernel's own leaky-ReLU branches where float64's u is within TAU of zero, plain float64
# everywhere else (tests/synthesis_branch_oracle.py).  Measured on an H100: 1.27e-5 (rows <=
# 1.6e-5) and 1.78e-5 (rows <= 1.9e-5).  ``plain bar`` (None: none) holds it against plain float64
# too: 1.27e-5 on the first net, which borrows no branch; the second borrows 9 positions (|u64| <=
# 1.4e-5) and is 4.1e-3 from plain float64, each of its rows up to the one of the last flipped
# layer 0.7e-3 .. 5.4e-3 off -- the exact gradient of the network on the other branch.
GRAD_CASES = [((128, 128, 64, 32), 3, 5e-4, 3.5e-5), ((256, 128, 128, 96, 64), 2, None, 5e-5)]


@pytest.mark.parametrize('channels,batch,plain_bar,bar', GRAD_CASES)
def test_ws_grad_against_float64_autograd(cuda_lib, channels, batch, plain_bar, bar):
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    res = 4 << (len(channels) - 1)
    p = synthetic.make_synthesis_params(5, res, channels, 512, 'cuda')
    g = torch.Generator().manual_seed(8)
    ws = torch.randn(batch, 2 * len(channels), 512, generator=g).cuda()
    g_planes = torch.randn(batch, 3, res, res, 32, generator=g).cuda()
    w = ws.clone().requires_grad_()
    planes = FusedSynthesis.from_params(p).forward_differentiable(w, noise_mode='const')
    u_kernel = saved_preactivations(planes)
    planes.backward(g_planes)
    got = w.grad.double()
    # truth: autograd through the oracle in float64, the same upstream gradient channel-first
    print('\n%r B=%d' % (channels, batch))
    pd, wd, nz, masks, _ = BO.kernel_branches(p, u_kernel, ws, HS.const_noises(p))
    g_img = _cf(g_planes.double())
    want = BO.ws_grad(pd, wd, nz, g_img)
    want_br = BO.ws_grad(pd, wd, nz, g_img, masks)
    row, row_br = BO.row_errors(got, want), BO.row_errors(got, want_br)
    e, e_br = _rel(got, want), _rel(got, want_br)
    print('  ws.grad rel-L2 on the kernel\'s branches %.2e, per row %s' % (
        e_br, ' '.join('%.1e' % r for r in row_br)))
    print('  ws.grad rel-L2 vs plain float64 %.2e, per row %s' % (e, ' '.join('%.1e' % r for r in row)))
    assert e_br < bar, e_br
    assert max(row_br) < bar, row_br
    if plain_bar is not None:
        assert e < plain_bar, e
        assert max(row) < 2 * plain_bar, row


def test_out_of_scope_gradients_raise(cuda_lib):
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200.synthesis import FusedSynthesis
    p, ws, _, _ = HS.load_case(HS.CASES[0], 'cuda')
    fs = FusedSynthesis.from_params(p)
    with pytest.raises(_lib.NfiError):      # no CPU path
        fs.forward_differentiable(ws.cpu().requires_grad_())
    w = ws.clone().requires_grad_()
    planes = fs.forward_differentiable(w, noise_mode='const')
    (gw,) = torch.autograd.grad(planes.square().sum(), w, create_graph=False)
    assert torch.isfinite(gw).all()
    planes = fs.forward_differentiable(w, noise_mode='const')
    with pytest.raises(_lib.NfiError):      # a double backward (path length)
        torch.autograd.grad(planes.square().sum(), w, create_graph=True)
    p2 = dict(p)
    p2['b4.conv1.weight'] = p['b4.conv1.weight'].clone().requires_grad_()
    net = FusedSynthesis.from_params(p2).net
    net.parameters = lambda: [p2['b4.conv1.weight']]
    with pytest.raises(_lib.NfiError):      # weight gradients are not offered
        FusedSynthesis(net).forward_differentiable(w)


# full size on the kernel's branches, measured on an H100: 9.3e-5, against 3.2e-3 from plain float64
# (the module's own float64 and the oracle agree to 1e-15; 476 positions borrowed, |u64| <= 8e-5);
# the residual over the small nets' 2e-5 is the accumulation over K = 9 x 512
FULL_BAR = 2e-4
staged = pytest.mark.skipif(not RL.available(),
                            reason='reference not installed (oracle/stage_reference.py)')


@staged
def test_full_size_against_the_reference_module(cuda_lib):
    """512 channels, 256^2 planes, B = 2, eval, frozen: ws.grad against the module's own float64
    autograd; the module's eager fp32 error is printed next to ours.

    The forward's 1e-3 bar does not carry over: demodulation makes each layer's output nearly
    invariant to the scale of its style, so ds = sum_pos dx~ x - s (demodulation term) is a
    difference of two nearly equal sums.  Measured on an H100: the module's own eager fp32 leaves
    1.4e-3, the fused backward 3.2e-3.  The assert holds the fused backward within 5e-3 and within
    4x of the module's own fp32 error."""
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RL._import_reference()
    from models import stylegan
    torch.manual_seed(1234)
    net = stylegan.SynthesisNetwork(512, 256, 96).cuda().eval().requires_grad_(False)
    ws = torch.randn(2, net.num_ws, 512, device='cuda')
    g_planes = torch.randn(2, 3, 256, 256, 32, device='cuda') / 256
    w = ws.clone().requires_grad_()
    planes = FusedSynthesis(net).forward_differentiable(w)
    u_kernel = saved_preactivations(planes)
    planes.backward(g_planes)
    got = w.grad.double()
    w32 = ws.clone().requires_grad_()
    ref32 = torch.autograd.grad(net(w32), w32, _cf(g_planes))[0].double()
    net.double()
    wd = ws.double().requires_grad_()
    truth = torch.autograd.grad(net(wd), wd, _cf(g_planes.double()))[0]
    net.float()
    e_ours, e_ref = _rel(got, truth), _rel(ref32, truth)
    print('full-size ws.grad rel-L2 vs float64: fused %.3e, eager fp32 module %.3e' % (e_ours, e_ref))
    assert e_ours < 5e-3 and e_ours < 4 * e_ref, (e_ours, e_ref)
    # the oracle on the module's parameters (eval, noise_strength 0: no noise), on the kernel's
    # branches where float64's u is within TAU of zero
    pd, wd, nz, masks, _ = BO.kernel_branches(SO.extract_params(net), u_kernel, ws, tau=BO.TAU_FULL)
    g_img = _cf(g_planes.double())
    want = BO.ws_grad(pd, wd, nz, g_img)
    want_br = BO.ws_grad(pd, wd, nz, g_img, masks)
    e_plain, e_br = _rel(got, want), _rel(got, want_br)
    print('full-size ws.grad rel-L2: on the kernel\'s branches %.3e, plain float64 oracle %.3e '
          '(module %.3e)' % (e_br, e_plain, _rel(want, truth)))
    assert e_br < FULL_BAR, e_br


H = W = 32
S = 16


def _setup_generator(B=2, seed=1234):
    from nerf_from_image_b200 import render as R
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    torch.manual_seed(seed)
    g = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True,
                            disable_stylegan_noise=True).cuda().eval()
    g.requires_grad_(False)
    with torch.no_grad():
        g.decoder.net[2].bias[0] = -1.15            # a mask that is neither empty nor full
    cams = synthetic.make_cameras(seed, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    with torch.no_grad():
        ws = g.mapping_network(torch.randn(B, 512, device='cuda'), None)
    args = types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                 fine_sampling=True)
    R.configure(args, {'scene_range': cfg['scene_range'],
                       'white_background': cfg['white_background']})
    ref_render = RL.lift_render(cfg['scene_range'], cfg['white_background'], use_sdf=True,
                                attention_values=10, fine_sampling=True)
    return R, g, cams, ws, ref_render


@staged
@pytest.mark.parametrize('rows', [15, 1])
def test_inversion_step_through_render(cuda_lib, rows):
    """The inversion loop's step (run.py:1983-2309): latents and pose require grad, the generator
    is frozen; with ``enable_fused_inversion`` the planes and their backward run on the sm_90a
    synthesis kernels."""
    R, g, cams, ws, ref_render = _setup_generator()
    w0 = ws if rows == 15 else ws[:, :1].contiguous()
    res = []
    try:
        for fn, fused in ((ref_render, False), (R.render, True)):
            R.enable_fused_inversion(g, fused)
            w = w0.clone().requires_grad_()
            c2w = cams['c2w'].clone().requires_grad_()
            torch.manual_seed(41)
            out = fn(g, H, W, c2w, cams['focal'], None, cams['bbox'], w, S,
                     extra_model_outputs=['attention_values'])
            loss = out[0].square().mean() + out[2].mean() \
                + 0.1 * out[5]['attention_values'].square().mean()
            res.append((torch.autograd.grad(loss, [w, c2w]), torch.cuda.get_rng_state()))
    finally:
        R.enable_fused_inversion(g, False)
    ((gw_r, gc_r), s_r), ((gw_f, gc_f), s_f) = res
    assert torch.equal(s_r, s_f), 'RNG consumption differs'
    assert _rel(gw_f, gw_r) < 5e-3, _rel(gw_f, gw_r)
    assert _rel(gc_f, gc_r) < 5e-3, _rel(gc_f, gc_r)
    if rows == 15:   # the palette path: row 14 feeds the texture mapper only
        assert gw_r[:, 14].abs().sum() > 0
        assert _rel(gw_f[:, 14], gw_r[:, 14]) < 5e-3, _rel(gw_f[:, 14], gw_r[:, 14])


@staged
def test_trainable_synthesis_keeps_the_reference_module(cuda_lib):
    from nerf_from_image_b200 import generator as G
    from nerf_from_image_b200.synthesis import FusedSynthesis
    R, g, cams, ws, _ = _setup_generator()
    g.synthesis_network.b4.conv1.weight.requires_grad_(True)
    calls = []
    orig = FusedSynthesis.forward_differentiable
    FusedSynthesis.forward_differentiable = lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    R.enable_fused_inversion(g)
    try:
        w = ws.clone().requires_grad_()
        out = R.render(g, H, W, cams['c2w'], cams['focal'], None, cams['bbox'], w, S)
        out[0].mean().backward()
        assert not calls and w.grad is not None and w.grad.abs().sum() > 0
        assert g.synthesis_network.b4.conv1.weight.grad is not None
        assert not G.FusedInversionFront(g).supports(['sampler'], {})
        # frozen again: the fused path is taken
        g.synthesis_network.b4.conv1.weight.requires_grad_(False)
        w = ws.clone().requires_grad_()
        R.render(g, H, W, cams['c2w'], cams['focal'], None, cams['bbox'], w, S)[0].mean().backward()
        assert calls and w.grad.abs().sum() > 0
    finally:
        FusedSynthesis.forward_differentiable = orig
        R.enable_fused_inversion(g, False)
        g.requires_grad_(False)
