"""The fused LPIPS-VGG distance (nerf_from_image_b200/lpips.py, csrc/nfi_lpips.cu) on the GPU,
against the float64 oracle (oracle/lpips_oracle.py) on seeded random weights (lins |randn|) at 128^2:

1. distance and gradient at N = 64 (one GPU's share of a config-3 step) and N = 256, with the
   eager fp32 oracle's own error against float64 printed beside ours; the gradient on the kernel's
   ReLU / pool branches (read from its saved pre-activations), the plain-float64 figure printed;
2. the gradient to in1 as well (the inversion step's augmented targets require grad), and a
   non-square size whose deeper levels are 3 .. 20 positions wide;
3. an image with a constant region (exact positive pool ties);
4. relu5_3 zero everywhere: finite, zero contribution;
5. an image's distance and gradient are bit-identical alone and inside the batch;
6. the inversion step's closure through render.ParallelModel, in the plain form and in
   optimize_iter's (augmented copies, in1 requiring grad), against the float64 stand-in, beside the
   eager fp32 one;
7. the refusals."""
import copy
import types

import pytest
import torch

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.lpips import FusedLPIPS, saved_preactivations
from oracle import lpips_oracle as LO
from oracle import reference_lift as RL
from tests.lpips_standin import StandInLPIPSLoss, inversion_loss

pytestmark = pytest.mark.gpu

RES = 128
CHUNK = 16        # images per float64 oracle call
# Bars: distance relative error per image, gradient relative L2 on the kernel's branches, each also
# within 5x of the eager fp32 oracle's own error against float64.  Measured on an H100 (README 4.8):
# distance 4.6e-7 / 5.1e-7 at N = 64 / 256 (eager fp32 2.4e-7 / 3.0e-7), gradient 4.7e-5 (the
# eager fp32 gradient is 2-3e-3 from plain float64, as is ours: near-tied pool windows)
DIST_BAR, GRAD_BAR, EAGER_FACTOR = 1e-4, 1e-3, 5.0
NEAR_ABS = 1e-6   # near-identical pairs: |d - d64|; measured 1.9e-9 (eager fp32 1.9e-10)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _images(n, seed, device='cuda', h=RES, w=RES):
    g = torch.Generator().manual_seed(seed)
    # smooth structure plus pixel noise, in the [-1, 1] range of the inversion loss's inputs
    lo = torch.rand(n, 3, h // 8, w // 8, generator=g)
    x = torch.nn.functional.interpolate(lo, size=(h, w), mode='bilinear', align_corners=False)
    x = x + 0.1 * torch.randn(n, 3, h, w, generator=g)
    return (x * 2 - 1).clamp(-1, 1).to(device)


def _module(p):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return FusedLPIPS(StandInLPIPSLoss(p)).cuda()


def _fused(m, x, y):
    a = x.clone().requires_grad_()
    d = m(a, y)[:, 0]
    us = saved_preactivations(d)
    d.sum().backward()
    return d.detach(), a.grad, us


def _oracle(p, x, y, us=None, grad=True, grad1=False):
    """Chunked oracle distance and gradient (dtype of p); with ``us``, on those branches; with
    grad1, the gradient to y as well (returned as a pair)."""
    N, ds, gs, gs1 = x.shape[0], [], [], []
    for s in range(0, N, CHUNK):
        e = min(N, s + CHUNK)
        br0 = br1 = None
        if us is not None:
            br0 = LO.branches_from_u([u[s:e] for u in us])
            br1 = LO.branches_from_u([u[N + s:N + e] for u in us])
        a = x[s:e].to(p['shift'].dtype).requires_grad_(grad)
        b = y[s:e].to(a.dtype).requires_grad_(grad1)
        with torch.set_grad_enabled(grad):
            d = LO.distance(p, a, b, br0, br1)
            if grad1:
                ga, gb = torch.autograd.grad(d.sum(), [a, b])
                gs.append(ga.detach())
                gs1.append(gb.detach())
            elif grad:
                gs.append(torch.autograd.grad(d.sum(), a)[0].detach())
        ds.append(d.detach())
    if grad1:
        return torch.cat(ds), (torch.cat(gs), torch.cat(gs1))
    return torch.cat(ds), (torch.cat(gs) if grad else None)


def _check(p32, x, y, label, dist_rel=True):
    p64 = LO.to(p32, 'cuda', torch.float64)
    m = _module(LO.to(p32, 'cpu', torch.float32))
    d, g, us = _fused(m, x, y)
    d64, g64 = _oracle(p64, x, y)
    d32, g32 = _oracle(LO.to(p32, 'cuda', torch.float32), x, y)
    _, g64b = _oracle(p64, x, y, us)
    if dist_rel:
        e_d = ((d.double() - d64).abs() / d64.abs()).max().item()
        e_d32 = ((d32.double() - d64).abs() / d64.abs()).max().item()
    else:
        e_d = (d.double() - d64).abs().max().item()
        e_d32 = (d32.double() - d64).abs().max().item()
    e_g, e_gp = _rel(g.double(), g64b), _rel(g.double(), g64)
    e_g32 = _rel(g32.double(), g64)
    print('%s: distance %s error %.2e (eager fp32 %.2e); gradient rel-L2 on the kernel\'s branches '
          '%.2e, plain float64 %.2e (eager fp32 %.2e)'
          % (label, 'rel' if dist_rel else 'abs', e_d, e_d32, e_g, e_gp, e_g32))
    assert torch.isfinite(d).all() and torch.isfinite(g).all()
    return e_d, e_d32, e_g, e_g32


@pytest.mark.parametrize('N', [64, 256])
def test_distance_and_gradient_against_float64(cuda_lib, N):
    p = LO.make_weights(seed=1)
    x, y = _images(N, seed=2), _images(N, seed=3)
    e_d, e_d32, e_g, e_g32 = _check(p, x, y, 'N=%d distinct pairs' % N)
    assert e_d < DIST_BAR and e_d < EAGER_FACTOR * max(e_d32, 1e-7), (e_d, e_d32)
    assert e_g < GRAD_BAR and e_g < EAGER_FACTOR * max(e_g32, 1e-7), (e_g, e_g32)


def test_gradient_to_both_inputs(cuda_lib):
    """in1 requiring grad (optimize_iter's augmented targets): one backward over both halves.  in0's
    gradient is bit-identical to the in0-only backward's; in1's is held to the same bars."""
    p = LO.make_weights(seed=21)
    N = 64
    x, y = _images(N, seed=22), _images(N, seed=23)
    m = _module(p)
    d0, g0_only, _ = _fused(m, x, y)
    a, b = x.clone().requires_grad_(), y.clone().requires_grad_()
    d = m(a, b)[:, 0]
    us = saved_preactivations(d)
    d.sum().backward()
    assert torch.equal(d.detach(), d0)
    assert torch.equal(a.grad, g0_only)
    p64 = LO.to(p, 'cuda', torch.float64)
    _, (g64_0, g64_1) = _oracle(p64, x, y, us, grad1=True)
    _, (g32_0, g32_1) = _oracle(LO.to(p, 'cuda', torch.float32), x, y, grad1=True)
    _, (p64_0, p64_1) = _oracle(p64, x, y, grad1=True)
    e0, e1 = _rel(a.grad.double(), g64_0), _rel(b.grad.double(), g64_1)
    e32 = _rel(g32_1.double(), p64_1)
    print('gradient to both inputs, rel-L2 on the kernel\'s branches: in0 %.2e, in1 %.2e; in1 against '
          'plain float64 %.2e (eager fp32 %.2e)' % (e0, e1, _rel(b.grad.double(), p64_1), e32))
    assert e0 < GRAD_BAR and e1 < GRAD_BAR, (e0, e1)
    assert e1 < EAGER_FACTOR * e32, (e1, e32)


def test_non_square_size(cuda_lib):
    """48 x 80: widths 80, 40, 20, 10, 5 and heights 48, 24, 12, 6, 3 at the five levels -- tiles
    that are mostly outside the image, on every side."""
    p = LO.make_weights(seed=24)
    x, y = _images(8, seed=25, h=48, w=80), _images(8, seed=26, h=48, w=80)
    e_d, e_d32, e_g, e_g32 = _check(p, x, y, '48 x 80')
    assert e_d < DIST_BAR and e_g < GRAD_BAR, (e_d, e_g)


def test_near_identical_pairs(cuda_lib):
    """in1 = in0 + 1e-3 noise: the distance is a sum of squares of nearly cancelling differences,
    so it is held to an absolute bound (NEAR_ABS) rather than a relative one."""
    p = LO.make_weights(seed=4)
    x = _images(16, seed=5)
    y = x + 1e-3 * torch.randn(x.shape, generator=torch.Generator().manual_seed(6)).cuda()
    e_d, _, e_g, e_g32 = _check(p, x, y, 'near-identical pairs', dist_rel=False)
    assert e_d < NEAR_ABS, e_d
    assert e_g < 10 * GRAD_BAR, (e_g, e_g32)


def test_constant_region_pool_ties(cuda_lib):
    p = LO.make_weights(seed=7)
    x, y = _images(8, seed=8), _images(8, seed=9)
    x[:, :, 16:80, 8:72] = 0.25          # a flat background: exact positive ties in the pools
    y[:, :, 40:120, 40:120] = -0.5
    m = _module(p)
    d, g, us = _fused(m, x, y)
    ties = 0
    for l in LO.POOLED:
        win = LO._windows(us[l][:8].clamp_min(0))
        top = win.max(dim=-1, keepdim=True).values
        ties += ((win == top).sum(-1) > 1).logical_and(top[..., 0] > 0).sum().item()
    assert ties > 1000, ties
    e_d, e_d32, e_g, e_g32 = _check(p, x, y, 'constant regions (%d tied windows)' % ties)
    assert e_d < DIST_BAR, e_d
    assert e_g < GRAD_BAR, e_g


def test_zero_tap_vectors_are_finite_and_contribute_nothing(cuda_lib):
    p = LO.make_weights(seed=10)
    p['conv_b'][12] = p['conv_b'][12] - 1e3        # relu5_3 = 0 at every position
    x, y = _images(4, seed=11), _images(4, seed=12)
    m = _module(p)
    d, g, us = _fused(m, x, y)
    assert us[12].max() < 0
    assert torch.isfinite(d).all() and torch.isfinite(g).all()
    p64 = LO.to(p, 'cuda', torch.float64)
    d64, g64 = _oracle(p64, x, y)
    # the same distance without the fifth tap: it contributes exactly nothing
    q = dict(p64, lin=p64['lin'][:4] + [torch.zeros_like(p64['lin'][4])])
    d64_4, _ = _oracle(q, x, y, grad=False)
    assert torch.equal(d64, d64_4)
    assert ((d.double() - d64).abs() / d64).max() < DIST_BAR
    assert _rel(g.double(), g64) < GRAD_BAR * 10


def test_an_image_alone_and_in_the_batch_are_bit_identical(cuda_lib):
    p = LO.make_weights(seed=13)
    m = _module(p)
    x, y = _images(64, seed=14), _images(64, seed=15)
    d, g, _ = _fused(m, x, y)
    for i in (0, 37, 63):
        di, gi, _ = _fused(m, x[i:i + 1], y[i:i + 1])
        assert torch.equal(di[0], d[i]), i
        assert torch.equal(gi[0], g[i]), i


def test_refusals(cuda_lib):
    m = _module(LO.make_weights(seed=16))
    x, y = _images(2, seed=17), _images(2, seed=18)
    with pytest.raises(_lib.NfiError):
        m(x[:, :, :120, :120], y[:, :, :120, :120])        # not a multiple of 16
    with pytest.raises(_lib.NfiError):
        m(x[:0], y[:0])                                      # no images
    with pytest.raises(_lib.NfiError):
        m(x)
    a = x.clone().requires_grad_()
    d = m(a, y).sum()
    d.backward(retain_graph=True)
    with pytest.raises(_lib.NfiError):
        d.backward()                                         # second backward
    a = x.clone().requires_grad_()
    with pytest.raises(_lib.NfiError):
        torch.autograd.grad(m(a, y).sum(), a, create_graph=True)   # double backward
    m.conv3_weight.requires_grad_(True)
    with pytest.raises(_lib.NfiError):
        m(x, y)                                              # a weight requires grad
    m.conv3_weight.requires_grad_(False)
    # normalize / reduction as the reference's LPIPSLoss
    x01, y01 = (x + 1) / 2, (y + 1) / 2
    assert torch.equal(m(x01, y01, normalize=True), m(2 * x01 - 1, 2 * y01 - 1))
    assert m(x, y, reduction='mean').shape == ()


# ---- the inversion step through ParallelModel (reference generator staged under oracle/_ref) ----
H = W = 32
S = 16
staged = pytest.mark.skipif(not RL.available(),
                            reason='reference not installed (oracle/stage_reference.py)')


@staged
@pytest.mark.parametrize('form', ['plain', 'optimize_iter'])
def test_inversion_closure_through_parallel_model(cuda_lib, form):
    """run.py's closure form: ParallelModel(..., lpips_net=FusedLPIPS(standin)) and the eager fp32
    stand-in, each against the stand-in in float64: the loss and the gradients of the latents and
    the pose.  'plain' calls lpips_net(pred, target); 'optimize_iter' builds the call as
    run.py:2211-2235 does (15 augmented copies of cat(pred, target), split again: in1 requires
    grad)."""
    from fixtures import synthetic
    from nerf_from_image_b200 import render as R
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    torch.manual_seed(1234)
    g = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True,
                            disable_stylegan_noise=True).cuda().eval()
    g.requires_grad_(False)
    B = 2
    cams = synthetic.make_cameras(1234, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    with torch.no_grad():
        ws = g.mapping_network(torch.randn(B, 512, device='cuda'), None)
    R.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                      fine_sampling=True),
                {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    R.depth_samples_per_ray = S
    standin = StandInLPIPSLoss(LO.make_weights(seed=19)).cuda()
    target = _images(B, seed=20)[:, :, :H, :W].contiguous()

    def closure(self_, rgb, mask, extra, model_outputs, target):
        pred = rgb.permute(0, 3, 1, 2) * 2 - 1
        dt = self_.lpips_net.lpips.scaling_layer.shift.dtype if hasattr(self_.lpips_net, 'lpips') \
            else torch.float32
        if form == 'plain':
            return self_.lpips_net(pred.to(dt), target.to(dt)).mean()
        return inversion_loss(self_.lpips_net, pred.to(dt), target.to(dt))

    res = []
    truth = copy.deepcopy(standin).double()
    for net in (truth, standin, FusedLPIPS(standin)):
        pm = R.ParallelModel(H, model=g, model_ema=g, lpips_net=net)
        w = ws.clone().requires_grad_()
        c2w = cams['c2w'].clone().requires_grad_()
        torch.manual_seed(41)
        loss = pm(c2w, cams['focal'], None, cams['bbox'], w, closure=closure,
                  closure_params={'target': target})
        res.append((loss.detach().double(), torch.autograd.grad(loss, [w, c2w])))
    (l_t, (gw_t, gc_t)), (l_r, (gw_r, gc_r)), (l_f, (gw_f, gc_f)) = res
    e = {k: (abs(l - l_t).item() / l_t.item(), _rel(gw.double(), gw_t.double()),
             _rel(gc.double(), gc_t.double()))
         for k, (l, (gw, gc)) in (('eager', res[1]), ('fused', res[2]))}
    print(form + ' closure vs the float64 stand-in: loss / ws.grad / c2w.grad rel error: fused %.2e %.2e %.2e, '
          'eager fp32 stand-in %.2e %.2e %.2e' % (e['fused'] + e['eager']))
    assert gw_t.abs().sum() > 0 and gc_t.abs().sum() > 0
    assert e['fused'][0] < DIST_BAR
    # the rendered image is the same in every arm; what differs is the loss's gradient to it, where
    # near-tied pool windows of the fp32 runs pick other maxima than float64's.  The eager error is
    # floored at 1e-3: over optimize_iter's 16 augmented copies the eager stand-in happened to land
    # at 2.3-2.8e-4 on ws, the fused loss at 1.1-1.3e-3 (measured on an H100, three runs; the render
    # and grid_sample backward accumulate with atomics, so the figures move between runs), both far
    # inside the 2-8e-3 that branch flips alone leave on one loss gradient (README 4.8)
    for i in (1, 2):
        assert e['fused'][i] < 2e-2 and e['fused'][i] < EAGER_FACTOR * max(e['eager'][i], 1e-3), e
