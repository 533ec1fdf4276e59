"""The path-length regulariser's double backward on sm_90a (``FusedSynthesis.
forward_trainable_with_path_length``: nfi_synthesis_backward for pl_grad, nfi_synthesis_backward_hvp
for its backward):

1. planes equal ``forward_trainable``'s and pl_grad equals ``nfi_synthesis_backward`` with
   g_planes = pl_noise, bit for bit;
2. every parameter group, ws and noise_strength against float64 double-backward autograd through
   the oracle on the kernel's own leaky-ReLU branches where float64's u is within TAU of zero
   (tests/synthesis_branch_oracle.py; lrelu'' = 0, so the masked double backward is defined);
3. a batch whose stacked GEMMs cover several waves of the persistent grid;
4. full size (512 channels, 256^2) against the module's own float64 double backward;
5. the G-step through ``render()`` with the path-length request, against the reference;
6. routing."""
import pytest
import torch

from oracle import reference_lift as RL
from oracle import synthesis_oracle as SO
from tests import helpers_synth as HS
from tests import synthesis_branch_oracle as BO
from tests import test_synthesis_param_grads_gpu as TP

pytestmark = pytest.mark.gpu

_rel, _cf, _trainable, _case, _const_raw = TP._rel, TP._cf, TP._trainable, TP._case, TP._const_raw


def _pl_noise(seed, B, R):
    """The draw forward_trainable_with_path_length makes after a seed (noise_mode 'const': no
    synthesis noise is drawn before it), channel-last."""
    torch.manual_seed(seed)
    return (torch.randn(B, 3, 32, R, R, device='cuda') / R).permute(0, 1, 3, 4, 2).contiguous()


def _fused_hvp(p, ws, t, seed=0, u_out=None):
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    pt = _trainable(p)
    w = ws.clone().requires_grad_()
    torch.manual_seed(seed)
    planes, pl_grad = FusedSynthesis.from_params(pt).forward_trainable_with_path_length(w, 'const')
    if u_out is not None:
        u_out += saved_preactivations(planes)
    (pl_grad * t).sum().backward()
    grads = {k: v.grad for k, v in pt.items() if torch.is_tensor(v) and v.grad is not None}
    return planes.detach(), pl_grad.detach(), w.grad, grads


def _float64_hvp(p, ws, n_cl, t, noises, masks=None):
    pd = {k: (v.double().requires_grad_() if torch.is_tensor(v) and v.is_floating_point() else v)
          for k, v in p.items()}
    wd = ws.detach().double().requires_grad_()
    nz = {k: raw.double() * pd[k + '.noise_strength'] for k, raw in noises.items()}
    img = SO.synthesis_forward(pd, wd, nz) if masks is None else BO.synthesis_forward(pd, wd, nz, masks)[0]
    (gws,) = torch.autograd.grad((img * _cf(n_cl.double())).sum(), wd, create_graph=True)
    for v in nz.values():
        v.retain_grad()
    (gws * t.double()).sum().backward()
    grads = {k: v.grad for k, v in pd.items() if torch.is_tensor(v) and v.grad is not None}
    grads['|terms|'] = {k: (nz[k].grad * raw.double()).abs().sum().item() for k, raw in noises.items()}
    return wd.grad, grads


def _errors(got_ws, got, want_ws, want):
    """-> {name: rel-L2} over every gradient float64 forms, plus 'ws'.  A noise_strength
    gradient is one sum of terms that largely cancel: its error is taken relative to the sum of
    their magnitudes, as in test_synthesis_param_grads_gpu.py."""
    want = dict(want)
    terms = want.pop('|terms|', {})
    errs = {'ws': _rel(got_ws.double(), want_ws)}
    for k, v in want.items():
        if k.endswith('.noise_strength'):
            errs[k] = abs(got[k].double() - v).item() / max(terms[k[:-len('.noise_strength')]], 1e-30)
        elif v.abs().sum() > 0:
            errs[k] = _rel(got[k].double(), v)
    return errs


def _hvp_case(channels, batch, seed=5):
    """-> (p, errors against float64 on the kernel's branches, errors against plain float64)"""
    p, ws, _ = _case(channels, batch, seed)
    R = p['meta']['img_resolution']
    t = torch.randn(ws.shape, generator=torch.Generator().manual_seed(9)).cuda()
    u_kernel = []
    _, _, g_ws, got = _fused_hvp(p, ws, t, u_out=u_kernel)
    print('\n%r B=%d' % (channels, batch))
    masks = BO.kernel_branches(p, u_kernel, ws, HS.const_noises(p))[3]
    out = []
    for what, m in (('the kernel\'s branches', masks), ('plain float64', None)):
        want_ws, want = _float64_hvp(p, ws, _pl_noise(0, batch, R), t, _const_raw(p), m)
        errs = _errors(g_ws, got, want_ws, want)
        worst = sorted(((e, k) for k, e in errs.items()), reverse=True)[:6]
        print('  HVP rel-L2 on %s: ws %.2e; worst %s' % (
            what, errs['ws'], ', '.join('%s %.1e' % (k, e) for e, k in worst)))
        out.append(errs)
    for r in p['meta']['resolutions']:   # the ToRGB bias does not enter <t, pl_grad>
        assert got['b%d.torgb.bias' % r].abs().max().item() == 0.0
    return p, out[0], out[1]


def test_planes_and_pl_grad_equal_the_first_order_entries(cuda_lib):
    from nerf_from_image_b200.synthesis import FusedSynthesis
    for channels, batch in (((128, 128, 64, 32), 3), ((64, 64, 32), 2)):
        p, ws, _ = _case(channels, batch)
        R = p['meta']['img_resolution']
        fs = FusedSynthesis.from_params(_trainable(p))
        torch.manual_seed(0)
        planes, pl_grad = fs.forward_trainable_with_path_length(ws.clone().requires_grad_(), 'const')
        plain = fs.forward_trainable(ws.clone().requires_grad_(), 'const')
        assert torch.equal(planes, plain)
        w = ws.clone().requires_grad_()
        FusedSynthesis.from_params(p).forward_differentiable(w, 'const').backward(_pl_noise(0, batch, R))
        assert torch.equal(pl_grad, w.grad), _rel(pl_grad.double(), w.grad.double())


# every group of the HVP (ws, weights, biases, affines, b4.const; noise_strength relative to the sum
# of its terms) against float64 on the kernel's own leaky-ReLU branches where float64's u is within
# TAU of zero, plain float64 elsewhere.  Measured on an H100, worst group: 1.7e-5 on (128,128,64,32)
# B=3 (no branch borrowed; the same against plain float64), 2.5e-5, 2.0e-5 and 2.6e-5 on the three
# nets below (against plain float64 9.3e-3, 5.5e-3, 7.1e-3), 1.8e-5 at B = 34 (1.5e-3 .. 3.6e-3
# against plain float64).
HVP_BAR = 5e-5


def test_hvp_against_float64_double_backward(cuda_lib):
    _, errs, plain = _hvp_case((128, 128, 64, 32), 3)
    bad = {k: e for k, e in errs.items() if not e < HVP_BAR}
    assert not bad, bad
    bad = {k: e for k, e in plain.items() if e > 1e-4}
    assert not bad, bad


NARROW = [((256, 128, 128, 96, 64), 2), ((64, 64, 64, 32, 32, 32, 32), 2),
          ((128, 128, 128, 64, 64, 64), 2)]


@pytest.mark.parametrize('channels,batch', NARROW)
def test_hvp_on_the_narrow_nets_at_the_flat_bar(cuda_lib, channels, batch):
    _, errs, _ = _hvp_case(channels, batch)
    bad = {k: e for k, e in errs.items() if not e < HVP_BAR}
    assert not bad, bad


def test_hvp_over_several_waves(cuda_lib):
    """Batch picked from the SM count: the stacked (2B-image) conv launches of the last block run
    at least two waves of the persistent grid and never a whole number of them."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = lambda b: 2 * b * 4            # 32x32 -> four 16x16 tiles, one 32-channel n-tile
    batch = next(b for b in range(2, 4 * sms) if tiles(b) >= 2 * sms and tiles(b) % sms)
    print('B=%d: %d tiles on %d SMs (%.2f waves)' % (batch, tiles(batch), sms, tiles(batch) / sms))
    _, errs, _ = _hvp_case((128, 128, 64, 32), batch)
    bad = {k: e for k, e in errs.items() if not e < HVP_BAR}
    assert not bad, bad


# full size on the kernel's branches, measured on an H100: every group 7.3e-5 .. 1.2e-4 (b4.const
# the worst), against 3.6e-3 .. 4.1e-3 from plain float64 (222 positions borrowed, |u64| <= 8e-5);
# the residual over the small nets' 2e-5 is the accumulation over K = 9 x 512
FULL_BAR = 3e-4


@pytest.mark.skipif(not RL.available(), reason='reference not installed (oracle/stage_reference.py)')
def test_full_size_against_the_reference_module(cuda_lib):
    """512 channels, 256^2 planes, B = 1: every group of the HVP against the module's own float64
    double backward.  Measured on an H100: fused 3.6e-3 .. 4.1e-3 against the eager fp32 module's
    0.9e-3 .. 1.25e-3, 3.2x .. 4.5x (ToRGB weight the worst: its tangent input carries the whole
    tangent-forward chain).  Bars: the first-order full-size test's 5e-3, and 5x the module."""
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RL._import_reference()
    from models import stylegan
    torch.manual_seed(1234)
    net = stylegan.SynthesisNetwork(512, 256, 96).cuda().eval().requires_grad_(True)
    B, R = 1, 256
    ws = torch.randn(B, net.num_ws, 512, device='cuda')
    t = torch.randn(B, net.num_ws, 512, device='cuda')
    names = [n for n, _ in net.named_parameters()]
    w = ws.clone().requires_grad_()
    torch.manual_seed(0)        # eval mode, noise_strength 0: no synthesis noise is drawn
    planes, pl_grad = FusedSynthesis(net).forward_trainable_with_path_length(w)
    u_kernel = saved_preactivations(planes)
    (pl_grad * t).sum().backward()
    got = [(q.grad if q.grad is not None else torch.zeros_like(q)).double()
           for q in net.parameters()] + [w.grad.double()]
    net.zero_grad(set_to_none=True)
    n_cf = _cf(_pl_noise(0, B, R))

    def module_hvp(dtype):
        wm = ws.to(dtype).requires_grad_()
        (g,) = torch.autograd.grad((net(wm) * n_cf.to(dtype)).sum(), wm, create_graph=True)
        return torch.autograd.grad((g * t.to(dtype)).sum(), list(net.parameters()) + [wm],
                                   allow_unused=True)
    ref32 = module_hvp(torch.float32)
    net.double()
    truth = module_hvp(torch.float64)
    net.float()

    def kind(n):
        for k in ('affine.weight', 'affine.bias', 'torgb.weight', 'const', 'noise_strength',
                  'weight', 'bias'):
            if n.endswith(k):
                return k
        return n
    groups = {}
    for n, a, r, tr in zip(names + ['ws'], got, ref32, truth):
        if tr is None or tr.abs().sum() == 0:
            continue
        groups.setdefault(kind(n), []).append((a.flatten(), r.double().flatten(), tr.flatten()))
    for k, trip in groups.items():
        a, r, tr = (torch.cat([x[i] for x in trip]) for i in range(3))
        e_ours, e_ref = _rel(a, tr), _rel(r, tr)
        print('full size HVP %-14s rel-L2 vs float64: fused %.3e, eager fp32 module %.3e'
              % (k, e_ours, e_ref))
        assert e_ours < 5e-3 and e_ours < 5 * e_ref, (k, e_ours, e_ref)
    # the oracle on the module's parameters (eval, noise_strength 0: no noise), on the kernel's
    # branches where float64's u is within TAU of zero
    p = SO.extract_params(net)
    masks = BO.kernel_branches(p, u_kernel, ws, tau=BO.TAU_FULL)[3]
    want_ws, want = _float64_hvp(p, ws, _pl_noise(0, B, R), t, _const_raw(p), masks)
    br = {}
    for n, a in zip(names + ['ws'], got):
        tr = want_ws if n == 'ws' else want.get(n)
        if tr is not None and tr.abs().sum() > 0:
            br.setdefault(kind(n), []).append((a.flatten(), tr.flatten()))
    for k, pairs in br.items():
        e = _rel(torch.cat([a for a, _ in pairs]), torch.cat([x for _, x in pairs]))
        print('full size HVP %-14s rel-L2 on the kernel\'s branches %.3e' % (k, e))
        assert e < FULL_BAR, (k, e)


# ---------------------------------------------------------------- through render()
staged = pytest.mark.skipif(not RL.available(),
                            reason='reference not installed (oracle/stage_reference.py)')
PL_REQUEST = ['sdf_eikonal_loss', 'total_variation_loss', 'entropy_loss', 'path_length']


@staged
def test_path_length_step_through_render(cuda_lib):
    from nerf_from_image_b200 import generator as G
    from tests import test_generator_step_gpu as TG
    R, g, cams, z, ref_render = TG._setup()
    calls = []
    orig = G.PathLengthGeneratorStepFront.__call__
    G.PathLengthGeneratorStepFront.__call__ = lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    res = []
    try:
        for fn, fused in ((ref_render, False), (R.render, True)):
            R.enable_fused_generator_step(g, fused)
            R.enable_fused_heads(g, fused)
            R.enable_fused_path_length(g, fused)
            torch.manual_seed(41)
            out = fn(g, TG.H, TG.W, cams['c2w'], cams['focal'], None, cams['bbox'], z, TG.S,
                     extra_model_outputs=list(PL_REQUEST))
            mo = out[5]
            ppl = mo['path_length']
            loss = out[0].square().mean() + (out[2] - 0.5).square().mean() \
                + 0.1 * mo['sdf_eikonal_loss'].mean() + mo['total_variation_loss'].mean() \
                + 0.01 * mo['entropy_loss'].mean() + 2.0 * (ppl - 0.5 * ppl.detach().mean()).square().mean()
            res.append((ppl.detach(), TG._grads(loss, g), torch.cuda.get_rng_state()))
    finally:
        G.PathLengthGeneratorStepFront.__call__ = orig
        R.enable_fused_generator_step(g, False)
        R.enable_fused_heads(g, False)
        R.enable_fused_path_length(g, False)
    (p_r, g_r, s_r), (p_f, g_f, s_f) = res
    assert calls == [1], 'the fused call takes the path-length front'
    assert torch.equal(s_r, s_f), 'RNG consumption differs'
    e = _rel(p_f, p_r)
    print('path_length rel-L2 %.2e (%s vs %s)' % (e, p_f.tolist(), p_r.tolist()))
    assert e < 1e-3, e
    TG._compare(g, g_f, g_r)


@staged
def test_routing(cuda_lib):
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200 import generator as G
    from nerf_from_image_b200.synthesis import FusedSynthesis
    from tests import test_generator_step_gpu as TG
    R, g, cams, z, _ = TG._setup()
    front = G.PathLengthGeneratorStepFront(g)
    assert front.supports(['sampler'] + PL_REQUEST, {})
    assert not front.supports(['sampler'] + TG.HEADS, {})              # no path_length: G-step front's
    assert not front.supports(['sampler', 'path_length'], {'unknown_input': 1})
    with torch.no_grad():
        assert not front.supports(['sampler', 'path_length'], {})
    g.synthesis_network.requires_grad_(False)
    assert not front.supports(['sampler', 'path_length'], {})
    g.synthesis_network.requires_grad_(True)
    with pytest.raises(_lib.NfiError):
        front(None, z, ['sampler'])
    calls = []
    orig = FusedSynthesis.forward_trainable_with_path_length
    FusedSynthesis.forward_trainable_with_path_length = \
        lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    a = (g, TG.H, TG.W, cams['c2w'], cams['focal'], None, cams['bbox'], z, TG.S)
    try:
        R.enable_fused_generator_step(g)
        R.enable_fused_heads(g)
        R.render(*a, extra_model_outputs=['sdf_eikonal_loss', 'path_length'])
        assert not calls                                                 # not opted in
        R.enable_fused_path_length(g)
        out = R.render(*a, extra_model_outputs=['sdf_eikonal_loss', 'path_length'])
        assert calls == [1] and 'path_length' in out[5]
        out[5]['path_length'].sum().backward()
        R.render(*a, extra_model_outputs=list(TG.HEADS))[0].mean().backward()   # no path_length
        with torch.no_grad():
            R.render(*a)
        g.synthesis_network.requires_grad_(False)                        # frozen synthesis
        R.render(*a)[0].mean().backward()
        g.synthesis_network.requires_grad_(True)
        pm = R.ParallelModel(TG.H, model=g, model_ema=g)                 # pretrain_sdf
        pm(None, None, None, None, z, pretrain_sdf=True)['sdf_distance_loss'].mean().backward()
        assert calls == [1]
    finally:
        FusedSynthesis.forward_trainable_with_path_length = orig
        R.enable_fused_generator_step(g, False)
        R.enable_fused_heads(g, False)
        R.enable_fused_path_length(g, False)


def test_out_of_scope_calls_raise(cuda_lib):
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200.synthesis import FusedSynthesis
    p, ws, _ = _case((64, 64, 32), 2)
    fs = FusedSynthesis.from_params(_trainable(p))
    w = ws.clone().requires_grad_()
    _, pl_grad = fs.forward_trainable_with_path_length(w, 'const')
    with pytest.raises(_lib.NfiError):      # a third derivative
        torch.autograd.grad(pl_grad.square().sum(), w, create_graph=True)
    _, pl_grad = fs.forward_trainable_with_path_length(w, 'const')
    loss = pl_grad.square().sum()
    loss.backward(retain_graph=True)
    with pytest.raises(_lib.NfiError):      # a second backward on one forward
        loss.backward()
