"""The synthesis backward to the parameters on sm_90a (nfi_synthesis_forward_saved +
nfi_synthesis_backward_params through ``FusedSynthesis.forward_trainable``):

1. the trainable forward emits exactly the plain forward's planes, and its ws.grad equals the
   latents-only backward's bit for bit;
2. the weight-gradient GEMM on its own: the last block's ToRGB and conv1 gradients, which depend
   only on the planes' gradient, the saved forward and the K = 96 ToRGB data gradient, against
   float64 autograd with tight bars;
3. every parameter group, per block, against float64 autograd through the oracle on the kernel's
   own leaky-ReLU branches where float64's u is within TAU of zero (tests/synthesis_branch_oracle
   .py), on the two nets of test_synthesis_backward_gpu.py and two narrow nets;
4. a net whose weight GEMM covers more than two waves of work items, never a whole number;
5. noise_strength == 0 in training mode still receives its gradient;
6. the entry raises on a CPU tensor, a double backward and a second backward."""
import math

import pytest
import torch

from fixtures import synthetic
from oracle import synthesis_oracle as SO
from tests import helpers_synth as HS
from tests import synthesis_branch_oracle as BO

pytestmark = pytest.mark.gpu

GROUPS = ('weight', 'bias', 'affine.weight', 'affine.bias')


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _cf(planes_cl):
    from nerf_from_image_b200.synthesis import planes_channel_first
    return planes_channel_first(planes_cl)


def _trainable(p):
    """A copy of the parameter dict whose float tensors require grad."""
    return {k: (v.clone().requires_grad_() if torch.is_tensor(v) and v.is_floating_point() else v)
            for k, v in p.items()}


def _layer_keys(p):
    keys = []
    for r in p['meta']['resolutions']:
        for name in ('conv0', 'conv1', 'torgb'):
            pre = 'b%d.%s' % (r, name)
            if pre + '.weight' in p:
                keys.append(pre)
    return keys


def _fused_grads(p, ws, g_planes, noise_mode='const', training=False, u_out=None):
    """``u_out``: a list that receives the saved forward's pre-activations."""
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    pt = _trainable(p)
    w = ws.clone().requires_grad_()
    planes = FusedSynthesis.from_params(pt, training=training).forward_trainable(w, noise_mode)
    if u_out is not None:
        u_out += saved_preactivations(planes)
    planes.backward(g_planes)
    grads = {k: v.grad for k, v in pt.items() if torch.is_tensor(v) and v.grad is not None}
    return planes.detach(), w.grad, grads


def _float64_grads(p, ws, g_planes, noises, masks=None):
    """Autograd through the oracle in float64.  ``noises``: {layer: raw [B or 1,1,res,res]} to be
    multiplied by the layer's noise_strength (so noise_strength gets its gradient); ``masks``: the
    leaky-ReLU branches (tests/synthesis_branch_oracle.py), None for the oracle's own."""
    pd = {k: (v.double().requires_grad_() if torch.is_tensor(v) and v.is_floating_point() else v)
          for k, v in p.items()}
    wd = ws.double().requires_grad_()
    nz = {k: raw.double() * pd[k + '.noise_strength'] for k, raw in noises.items()}
    for v in nz.values():
        v.retain_grad()
    img = SO.synthesis_forward(pd, wd, nz) if masks is None else BO.synthesis_forward(pd, wd, nz, masks)[0]
    img.backward(_cf(g_planes.double()))
    grads = {k: v.grad for k, v in pd.items() if torch.is_tensor(v) and v.grad is not None}
    # noise_strength.grad = sum_{b,p} g_noise raw: the magnitude of its terms (its conditioning)
    grads['|terms|'] = {k: (nz[k].grad * raw.double()).abs().sum().item() for k, raw in noises.items()}
    return wd.grad, grads


def _const_raw(p):
    return {k: p[k + '.noise_const'][None, None] for k, info in p['meta']['layers'].items()
            if info['use_noise'] and float(p[k + '.noise_strength']) != 0.0}


def _case(channels, batch, seed=5):
    res = 4 << (len(channels) - 1)
    p = synthetic.make_synthesis_params(seed, res, channels, 512, 'cuda')
    g = torch.Generator().manual_seed(8)
    ws = torch.randn(batch, 2 * len(channels), 512, generator=g).cuda()
    g_planes = torch.randn(batch, 3, res, res, 32, generator=g).cuda()
    return p, ws, g_planes


def _report(p, got, want, got_ws, want_ws):
    """-> {group: rel-L2} over all layers, and prints per layer."""
    lines, errs = [], {}
    for key in _layer_keys(p):
        row = []
        for grp in GROUPS:
            name = key + '.' + grp
            e = _rel(got[name].double(), want[name])
            errs[name] = e
            row.append('%s %.1e' % (grp, e))
        ns = key + '.noise_strength'
        if ns in want:
            errs[ns] = abs(got[ns].double() - want[ns]).item() / max(abs(want[ns]).item(), 1e-30)
            row.append('noise_strength %.1e' % errs[ns])
        lines.append('  %-10s %s' % (key, ', '.join(row)))
    c = 'b4.const'
    errs[c] = _rel(got[c].double(), want[c])
    errs['ws'] = _rel(got_ws.double(), want_ws)
    lines.append('  b4.const %.1e, ws %.1e' % (errs[c], errs['ws']))
    print('\n'.join(lines))
    return errs


def test_planes_and_ws_grad_equal_the_latents_only_entry(cuda_lib):
    from nerf_from_image_b200.synthesis import FusedSynthesis
    cases = [HS.load_case(c, 'cuda')[:2] for c in HS.CASES]
    p, ws, _ = _case((128, 128, 64, 32), 3)
    cases.append((p, ws))
    for p, ws in cases:
        res = p['meta']['img_resolution']
        g_planes = torch.randn(ws.shape[0], 3, res, res, 32,
                               generator=torch.Generator().manual_seed(3)).cuda()
        fs = FusedSynthesis.from_params(p)
        with torch.no_grad():
            plain = fs(ws, noise_mode='const')
        w = ws.clone().requires_grad_()
        fs.forward_differentiable(w, noise_mode='const').backward(g_planes)
        planes, g_ws, _ = _fused_grads(p, ws, g_planes)
        assert torch.equal(planes, plain)
        # bit for bit where act_backward_kernel's sums have one block per image (res <= 32: the
        # atomics then add onto zero in a fixed order)
        assert torch.equal(g_ws, w.grad), _rel(g_ws.double(), w.grad.double())


def test_last_block_weight_gemm_against_float64(cuda_lib):
    """The last block's ToRGB weight / bias and conv1 weight see only the planes' gradient, the
    saved forward and the K = 96 ToRGB data gradient -- the new GEMM's own accuracy.  Measured on
    an H100: ToRGB weight 1.5e-5 and 1.9e-5 (the bf16 pair keeps 16 of dimg's 24 bits), ToRGB
    bias 3.3e-7 and 3.9e-7, conv1 weight 1.7e-5 on (128,128,64,32).  On (256,128,128,96,64) the
    last conv1 weight is 7.9e-4 from plain float64: that net's forward takes the other leaky-ReLU
    branch than float64 at a few positions within rounding of zero, so it is held against float64
    on the kernel's branches in test_every_parameter_group_against_float64 instead."""
    for channels, batch in (((128, 128, 64, 32), 3), ((256, 128, 128, 96, 64), 2)):
        p, ws, g_planes = _case(channels, batch)
        _, _, got = _fused_grads(p, ws, g_planes)
        _, want = _float64_grads(p, ws, g_planes, _const_raw(p))
        last = 'b%d' % p['meta']['img_resolution']
        e_rw = _rel(got[last + '.torgb.weight'].double(), want[last + '.torgb.weight'])
        e_rb = _rel(got[last + '.torgb.bias'].double(), want[last + '.torgb.bias'])
        e_cw = _rel(got[last + '.conv1.weight'].double(), want[last + '.conv1.weight'])
        print('%r B=%d last block: torgb.weight %.2e torgb.bias %.2e conv1.weight %.2e'
              % (channels, batch, e_rw, e_rb, e_cw))
        assert e_rw < 3e-5 and e_rb < 1e-6, (e_rw, e_rb)
        if channels == (128, 128, 64, 32):
            assert e_cw < 1e-4, e_cw


def _grad_case(channels, batch):
    """-> (p, fused grads, ws.grad, {'plain': (truth, ws truth), 'branches': (...)})"""
    p, ws, g_planes = _case(channels, batch)
    u_kernel = []
    _, g_ws, got = _fused_grads(p, ws, g_planes, u_out=u_kernel)
    print('\n%r B=%d' % (channels, batch))
    masks = BO.kernel_branches(p, u_kernel, ws, HS.const_noises(p))[3]
    truths = {}
    for kind, m in (('plain', None), ('branches', masks)):
        want_ws, want = _float64_grads(p, ws, g_planes, _const_raw(p), m)
        print('rel-L2 against float64 on %s; ws rows %s' % (
            'the kernel\'s branches' if m else 'its own branches',
            ' '.join('%.1e' % r for r in BO.row_errors(g_ws.double(), want_ws))))
        truths[kind] = (want, want_ws)
    return p, got, g_ws, truths


def _group_errors(p, got, g_ws, want, want_ws):
    """_report, with noise_strength.grad taken relative to the sum of its terms' magnitudes (it is
    one sum of g_noise x noise over every position, whose terms largely cancel)."""
    errs = _report(p, got, want, g_ws, want_ws)
    for name in errs:
        if name.endswith('noise_strength'):
            layer = name[:-len('.noise_strength')]
            errs[name] = abs(got[name].double() - want[name]).item() / want['|terms|'][layer]
    return errs


# (channels, batch, plain bar): every group within GROUP_BAR (noise_strength: NOISE_BAR) of float64
# on the kernel's own leaky-ReLU branches where float64's u is within TAU of zero, plain float64
# elsewhere; ToRGB groups (whose gradients do not go through the data-gradient chain) within 1e-4
# of plain float64 on every net; every group within ``plain bar`` of plain float64 where set.
# Measured on an H100, worst group on the kernel's branches: 2.0e-5, 2.7e-5, 3.0e-5, 2.5e-5; against
# plain float64 2.0e-5 on the first net (no branch borrowed) and 7.3e-3, 5.0e-3, 1.0e-2 on the
# others (9, 36 and 18 positions borrowed); ToRGB groups <= 2.1e-5 against both.
GRAD_BARS = [((128, 128, 64, 32), 3, 5e-4), ((256, 128, 128, 96, 64), 2, None),
             ((64, 64, 64, 32, 32, 32, 32), 2, None), ((128, 128, 128, 64, 64, 64), 2, None)]
GROUP_BAR = 6e-5
NOISE_BAR = 3e-5   # measured: noise_strength <= 1.1e-5 of the sum of its terms' magnitudes


@pytest.mark.parametrize('channels,batch,plain_bar', GRAD_BARS)
def test_every_parameter_group_against_float64(cuda_lib, channels, batch, plain_bar):
    """Every weight, bias, affine and noise_strength group, b4.const and ws."""
    p, got, g_ws, truths = _grad_case(channels, batch)
    print('on the kernel\'s branches:')
    errs = _group_errors(p, got, g_ws, *truths['branches'])
    print('plain float64:')
    plain = _group_errors(p, got, g_ws, *truths['plain'])
    print('noise_strength (relative to the sum of its terms) on the kernel\'s branches: %s' % ', '.join(
        '%s %.1e' % (k, v) for k, v in errs.items() if k.endswith('noise_strength')))
    bad = {k: v for k, v in errs.items() if not v < (NOISE_BAR if k.endswith('noise_strength') else GROUP_BAR)}
    assert not bad, bad
    bad = {k: v for k, v in plain.items() if '.torgb.' in k and not v < 1e-4}
    assert not bad, bad
    if plain_bar is not None:
        bad = {k: v for k, v in plain.items() if not v < plain_bar}
        assert not bad, bad


def _wgrad_items(cout, cin, taps, batch, dom):
    """wgrad_tc_kernel's work items for one layer (plan_wgrad in csrc/nfi_synth.cu)."""
    kt_total = batch * math.ceil(dom / 4) * math.ceil(dom / 16)
    base = math.ceil(cout / 64) * math.ceil(cin / 64) * taps
    n_split = max(1, min(math.ceil(1024 / base), math.ceil(kt_total / 16)))
    split_len = math.ceil(kt_total / n_split)
    return base * math.ceil(kt_total / split_len)


def test_weight_gemm_over_several_waves(cuda_lib):
    """Batch picked from the SM count: the last conv1's work items cover at least two waves of
    the persistent grid (two CTAs per SM) and never a whole number of them."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = 2 * sms
    channels = (256, 256, 256, 256)
    for batch in range(2, 64):
        items = _wgrad_items(256, 256, 9, batch, 32)
        if items >= 2 * grid and items % grid:
            break
    items = _wgrad_items(256, 256, 9, batch, 32)
    assert items >= 2 * grid and items % grid, (items, grid)
    print('B=%d: %d work items on a grid of %d CTAs (%.2f waves)' % (batch, items, grid, items / grid))
    p, ws, g_planes = _case(channels, batch)
    _, _, got = _fused_grads(p, ws, g_planes)
    _, want = _float64_grads(p, ws, g_planes, _const_raw(p))
    # bars from the H100 measurement: conv1 weight 6.6e-4 (its demodulation term nearly cancels
    # the GEMM, as on the second net of the last-block test)
    for name, bar in (('b32.torgb.weight', 3e-5), ('b32.torgb.bias', 1e-6), ('b32.conv1.weight', 1e-3)):
        e = _rel(got[name].double(), want[name])
        print('%s rel-L2 %.2e' % (name, e))
        assert e < bar, (name, e)


def test_zero_noise_strength_gets_its_gradient_in_training(cuda_lib):
    channels, batch = (128, 64, 32), 2
    p, ws, g_planes = _case(channels, batch)
    for k, info in p['meta']['layers'].items():
        p[k + '.noise_strength'] = torch.zeros((), device='cuda')
    torch.manual_seed(77)
    _, _, got = _fused_grads(p, ws, g_planes, noise_mode='random', training=True)
    # the same draws, in the same order: one randn([B,1,res,res]) per noisy layer
    torch.manual_seed(77)
    raw = {}
    for r in p['meta']['resolutions']:
        for name in ('conv0', 'conv1'):
            k = 'b%d.%s' % (r, name)
            if k in p['meta']['layers']:
                raw[k] = torch.randn([batch, 1, r, r], device='cuda')
    _, want = _float64_grads(p, ws, g_planes, raw)
    for k in raw:
        g, t = got[k + '.noise_strength'].item(), want[k + '.noise_strength'].item()
        print('%s noise_strength.grad fused %.6e float64 %.6e' % (k, g, t))
        assert t != 0 and abs(g - t) < 1e-4 * abs(t), (k, g, t)


def test_out_of_scope_calls_raise(cuda_lib):
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200.synthesis import FusedSynthesis
    p, ws, _, _ = HS.load_case(HS.CASES[0], 'cuda')
    pt = _trainable(p)
    fs = FusedSynthesis.from_params(pt)
    with pytest.raises(_lib.NfiError):      # no CPU path
        fs.forward_trainable(ws.cpu().requires_grad_())
    w = ws.clone().requires_grad_()
    planes = fs.forward_trainable(w, noise_mode='const')
    with pytest.raises(_lib.NfiError):      # a double backward (path length)
        torch.autograd.grad(planes.square().sum(), w, create_graph=True)
    planes = fs.forward_trainable(w, noise_mode='const')
    loss = planes.square().sum()
    loss.backward(retain_graph=True)
    with pytest.raises(_lib.NfiError):      # a second backward on one forward
        loss.backward()
    # the other entries keep refusing trainable parameters
    net = fs.net
    net.parameters = lambda: [pt['b4.conv1.weight']]
    with pytest.raises(_lib.NfiError):
        FusedSynthesis(net)(ws)
    with pytest.raises(_lib.NfiError):
        FusedSynthesis(net).forward_differentiable(w)


# full size on the kernel's branches, measured on an H100: every group <= 9.3e-5 (ToRGB weight
# 6.5e-5, its bf16 pairs; ToRGB bias 2.8e-7), against 3.1e-3 .. 3.6e-3 from plain float64
FULL_BAR = 2e-4
staged = pytest.mark.skipif(not __import__('oracle.reference_lift', fromlist=['x']).available(),
                            reason='reference not installed (oracle/stage_reference.py)')


@staged
def test_full_size_against_the_reference_module(cuda_lib):
    """512 channels, 256^2 planes, B = 2, trainable: every parameter group against the module's
    own float64 autograd, within 5e-3 and within 4x of the module's eager fp32 error."""
    from oracle import reference_lift as RL
    from nerf_from_image_b200.synthesis import FusedSynthesis, saved_preactivations
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RL._import_reference()
    from models import stylegan
    torch.manual_seed(1234)
    net = stylegan.SynthesisNetwork(512, 256, 96).cuda().eval().requires_grad_(True)
    ws = torch.randn(2, net.num_ws, 512, device='cuda')
    g_planes = torch.randn(2, 3, 256, 256, 32, device='cuda') / 256
    names = [n for n, _ in net.named_parameters()]
    w = ws.clone().requires_grad_()
    planes = FusedSynthesis(net).forward_trainable(w)
    u_kernel = saved_preactivations(planes)
    planes.backward(g_planes)
    got = [(q.grad if q.grad is not None else torch.zeros_like(q)).double()
           for q in net.parameters()] + [w.grad.double()]
    net.zero_grad(set_to_none=True)
    w32 = ws.clone().requires_grad_()
    ref32 = torch.autograd.grad(net(w32), list(net.parameters()) + [w32], _cf(g_planes),
                                allow_unused=True)
    net.double()
    wd = ws.double().requires_grad_()
    truth = torch.autograd.grad(net(wd), list(net.parameters()) + [wd], _cf(g_planes.double()),
                                allow_unused=True)
    net.float()

    def kind(n):
        for k in ('affine.weight', 'affine.bias', 'torgb.weight', 'torgb.bias', 'const',
                  'noise_strength', 'weight', 'bias'):
            if n.endswith(k):
                return k
        return n
    groups = {}
    for n, a, r, t in zip(names + ['ws'], got, ref32, truth):
        if t is None or t.abs().sum() == 0:
            continue
        groups.setdefault(kind(n), []).append((a.flatten(), r.double().flatten(), t.flatten()))
    for k, trip in groups.items():
        a, r, t = (torch.cat([x[i] for x in trip]) for i in range(3))
        e_ours, e_ref = _rel(a, t), _rel(r, t)
        print('full size %-14s rel-L2 vs float64: fused %.3e, eager fp32 module %.3e' % (k, e_ours, e_ref))
        if k == 'torgb.weight':
            # bf16-pair operands keep 16 significant bits: measured 6.5e-5 on an H100, against
            # the module's 1.5e-6; held to the bar of the small nets' ToRGB groups
            assert e_ours < 1e-4, (k, e_ours, e_ref)
        else:
            assert e_ours < 5e-3 and e_ours < 4 * e_ref, (k, e_ours, e_ref)
    # the oracle on the module's parameters (eval, noise_strength 0: no noise), on the kernel's
    # branches where float64's u is within TAU of zero
    p = SO.extract_params(net)
    masks = BO.kernel_branches(p, u_kernel, ws, tau=BO.TAU_FULL)[3]
    want_ws, want = _float64_grads(p, ws, g_planes, _const_raw(p), masks)
    br = {}
    for n, a in zip(names + ['ws'], got):
        t = want_ws if n == 'ws' else want.get(n)
        if t is not None and t.abs().sum() > 0:
            br.setdefault(kind(n), []).append((a.flatten(), t.flatten()))
    for k, pairs in br.items():
        e = _rel(torch.cat([a for a, _ in pairs]), torch.cat([t for _, t in pairs]))
        print('full size %-14s rel-L2 on the kernel\'s branches %.3e' % (k, e))
        assert e < FULL_BAR, (k, e)
