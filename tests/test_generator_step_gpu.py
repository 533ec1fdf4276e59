"""The GAN generator step with the plane producer on sm_90a (``render.enable_fused_generator_step``
+ ``enable_fused_heads``) against the reference render + module: the reference ``Generator`` in
``train()`` mode with random synthesis noise, every generator parameter trainable.

1. the G-step through ``render()`` with the regulariser heads: the gradient of every generator
   parameter group (mapping, texture mapper, synthesis, decoder, beta), RNG consumption, and the
   dual discriminator's second call (['sampler'] only);
2. the same for ``ParallelModel``'s ``pretrain_sdf`` branch;
3. routing: 'path_length', ``no_grad`` and a frozen synthesis network keep their routes, and the
   front raises outside its envelope."""
import types

import pytest
import torch

from oracle import reference_lift as RL

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not RL.available(),
                                 reason='reference not installed (oracle/stage_reference.py)')]

H = W = 32
S = 16
HEADS = ['sdf_eikonal_loss', 'total_variation_loss', 'entropy_loss']


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _setup(B=2, seed=1234):
    from fixtures import synthetic
    from nerf_from_image_b200 import render as R
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    torch.manual_seed(seed)
    g = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True).cuda()
    with torch.no_grad():
        g.decoder.net[2].bias[0] = -1.15            # a mask that is neither empty nor full
    g.train().requires_grad_(True)
    cams = synthetic.make_cameras(seed, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    z = torch.randn(B, 512, device='cuda')
    args = types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                 fine_sampling=True)
    R.configure(args, {'scene_range': cfg['scene_range'],
                       'white_background': cfg['white_background']})
    ref_render = RL.lift_render(cfg['scene_range'], cfg['white_background'], use_sdf=True,
                                attention_values=10, fine_sampling=True)
    return R, g, cams, z, ref_render


def _groups(g):
    return {'mapping': list(g.mapping_network.parameters()),
            'texture_mapper': list(g.texture_mapper.parameters()),
            'synthesis': list(g.synthesis_network.parameters()),
            'decoder': list(g.decoder.parameters()),
            'beta': [g.beta]}


def _compare(g, grads_f, grads_r, bar=5e-3):
    names = [n for n, p in g.named_parameters()]
    worst = sorted(((_rel(a, b), n) for n, a, b in zip(names, grads_f, grads_r)
                    if b is not None and b.abs().sum() > 0), reverse=True)[:5]
    print('worst parameters:', ', '.join('%s %.1e' % (n, e) for e, n in worst))
    by_name = dict(zip(names, zip(grads_f, grads_r)))
    pid = {id(p): n for n, p in g.named_parameters()}
    for grp, ps in _groups(g).items():
        pairs = [by_name[pid[id(p)]] for p in ps if by_name[pid[id(p)]][1] is not None]
        if not pairs:        # not reached by this call (the texture mapper in SDF pre-training)
            assert all(by_name[pid[id(p)]][0] is None for p in ps), grp
            continue
        a = torch.cat([x.flatten() for x, _ in pairs])
        b = torch.cat([y.flatten() for _, y in pairs])
        e = _rel(a, b)
        print('%-15s rel-L2 %.2e' % (grp, e))
        assert b.abs().sum() > 0, grp
        assert e < bar, (grp, e)


def _grads(loss, g):
    return torch.autograd.grad(loss, list(g.parameters()), allow_unused=True)


def test_generator_step_through_render(cuda_lib):
    from nerf_from_image_b200 import generator as G
    R, g, cams, z, ref_render = _setup()
    calls = []
    orig = G.GeneratorStepFront.__call__
    G.GeneratorStepFront.__call__ = lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    res = []
    try:
        for fn, fused in ((ref_render, False), (R.render, True)):
            R.enable_fused_generator_step(g, fused)
            R.enable_fused_heads(g, fused)
            torch.manual_seed(41)
            out = fn(g, H, W, cams['c2w'], cams['focal'], None, cams['bbox'], z, S,
                     extra_model_outputs=list(HEADS))
            mo = out[5]
            loss = out[0].square().mean() + (out[2] - 0.5).square().mean() \
                + 0.1 * mo['sdf_eikonal_loss'].mean() + mo['total_variation_loss'].mean() \
                + 0.01 * mo['entropy_loss'].mean()
            g1 = _grads(loss, g)
            # the dual discriminator's second call: the render alone
            out = fn(g, H, W, cams['c2w'], cams['focal'], None, cams['bbox'], z, S)
            g2 = _grads(out[0].square().mean() + out[2].mean(), g)
            res.append((g1, g2, torch.cuda.get_rng_state()))
    finally:
        G.GeneratorStepFront.__call__ = orig
        R.enable_fused_generator_step(g, False)
        R.enable_fused_heads(g, False)
    (g1_r, g2_r, s_r), (g1_f, g2_f, s_f) = res
    assert len(calls) == 2, 'both fused calls take the generator-step front'
    assert torch.equal(s_r, s_f), 'RNG consumption differs'
    print('G-step with heads:')
    _compare(g, g1_f, g1_r)
    print('second call, sampler only:')
    _compare(g, g2_f, g2_r)


def test_pretrain_sdf_branch(cuda_lib):
    from nerf_from_image_b200 import generator as G
    R, g, cams, z, _ = _setup()
    pm = R.ParallelModel(H, model=g, model_ema=g)
    calls = []
    orig = G.GeneratorStepFront.__call__
    G.GeneratorStepFront.__call__ = lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    res = []
    try:
        for fused in (False, True):
            R.enable_fused_generator_step(g, fused)
            R.enable_fused_heads(g, fused)
            torch.manual_seed(3)
            out = pm(None, None, None, None, z, pretrain_sdf=True)
            loss = out['sdf_distance_loss'].mean() + 0.1 * out['sdf_eikonal_loss'].mean()
            res.append((out, _grads(loss, g), torch.cuda.get_rng_state()))
    finally:
        G.GeneratorStepFront.__call__ = orig
        R.enable_fused_generator_step(g, False)
        R.enable_fused_heads(g, False)
    (o_r, g_r, s_r), (o_f, g_f, s_f) = res
    assert calls == [1]
    assert torch.equal(s_r, s_f), 'RNG consumption differs'
    for k in ('sdf_distance_loss', 'sdf_eikonal_loss'):
        assert _rel(o_f[k], o_r[k]) < 1e-3, k
    _compare(g, g_f, g_r)


def test_routing(cuda_lib):
    from nerf_from_image_b200 import _lib
    from nerf_from_image_b200 import generator as G
    from nerf_from_image_b200.synthesis import FusedSynthesis
    R, g, cams, z, _ = _setup()
    front = G.GeneratorStepFront(g)
    assert front.supports(['sampler'] + HEADS, {})
    assert not front.supports(['sampler', 'path_length'], {})          # double backward
    assert not front.supports(['sampler'], {'unknown_input': 1})
    with torch.no_grad():
        assert not front.supports(['sampler'], {})                      # no_grad front's
    g.synthesis_network.requires_grad_(False)
    assert not front.supports(['sampler'], {})                          # inversion front's
    g.synthesis_network.requires_grad_(True)
    with pytest.raises(_lib.NfiError):
        front(None, z, ['sampler', 'path_length'])
    calls = []
    orig = FusedSynthesis.forward_trainable
    FusedSynthesis.forward_trainable = lambda self, *a, **k: calls.append(1) or orig(self, *a, **k)
    a = (g, H, W, cams['c2w'], cams['focal'], None, cams['bbox'], z, S)
    try:
        R.enable_fused_generator_step(g)
        R.enable_fused_heads(g)
        # path_length keeps today's route: the heads front with the reference module
        out = R.render(*a, extra_model_outputs=['sdf_eikonal_loss', 'path_length'])
        assert not calls and 'path_length' in out[5]
        with torch.no_grad():                                           # no_grad: not this front
            R.render(*a)
        assert not calls
        g.synthesis_network.requires_grad_(False)                       # frozen synthesis
        R.render(*a)[0].mean().backward()
        assert not calls
        g.synthesis_network.requires_grad_(True)
        R.render(*a)[0].mean().backward()                               # inside: fused
        assert calls == [1]
        R.enable_fused_generator_step(g, False)                         # off: today's route
        R.render(*a)[0].mean().backward()
        assert calls == [1]
    finally:
        FusedSynthesis.forward_trainable = orig
        R.enable_fused_generator_step(g, False)
        R.enable_fused_heads(g, False)
