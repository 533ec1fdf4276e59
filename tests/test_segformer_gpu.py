"""The fused SegFormer backbone on the GPU against the float64 oracle fed the same drop-path scales:
the features and every parameter-gradient group (one group per layer kind and stage, e.g.
``block3.*.attn.q.weight``), as rel-L2, with eager fp32's error against the same float64 printed
beside each.  Also: the module's drop-path draws and the CUDA generator's state, determinism, batch
independence, no workspace kept under no_grad, and an Adam step through nn.DataParallel."""
import re

import pytest
import torch

from nerf_from_image_b200 import _lib
from nerf_from_image_b200 import segformer as FS
from oracle import segformer_oracle as SO
from tests import helpers as Hh
from tests.segformer_standin import load, make_segformer

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FEATURE_BAR = 5e-5
GRAD_BAR = 2e-4


def _group(name):
    return re.sub(r'\.\d+\.', '.*.', name)


def _groups(grads):
    out = {}
    for n, g in grads.items():
        out.setdefault(_group(n), []).append(g.double().flatten().cpu())
    return {k: torch.cat(v) for k, v in out.items()}


def _rel(a, b):
    return Hh.rel_l2(a.double().cpu(), b.double().cpu())


def _case(B, H, depths, out, seed, init='reference', train=True, stress=False):
    """(fused, eager fp32) errors against float64: features, and per gradient group."""
    p = SO.make_params(depths, out, seed, dtype=torch.float32, init=init, stress=stress)
    m = load(make_segformer(out, depths), p).to(DEV).train(train)
    x = torch.randn(B, 3, H, H, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
    g = torch.randn(B, out, H // 4, H // 4, generator=torch.Generator().manual_seed(seed + 2)).to(DEV)
    torch.manual_seed(seed + 3)
    scales = FS.drop_scales(m, B, DEV)
    # float64 oracle with those scales
    pd = {k: v.double().to(DEV).requires_grad_() for k, v in p.items()}
    sl = list(scales.double()) if scales is not None else None
    want = SO.forward(pd, depths, x.double(), sl)
    want.backward(g.double())
    # eager fp32 with those scales (TF32 off)
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    pe = {k: v.to(DEV).requires_grad_() for k, v in p.items()}
    eager = SO.forward(pe, depths, x, list(scales) if scales is not None else None)
    eager.backward(g)
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    # fused, drawing the same masks from the same seed
    FS.enable_fused_segformer(m)
    m.zero_grad(set_to_none=True)
    torch.manual_seed(seed + 3)
    feats = m(x)
    feats.backward(g)
    torch.cuda.synchronize()
    gf = _groups({n: t.grad for n, t in m.named_parameters()})
    gd = _groups({n: t.grad for n, t in pd.items()})
    ge = _groups({n: t.grad for n, t in pe.items()})
    res = {'features': (_rel(feats, want), _rel(eager, want))}
    for k in gd:
        res[k] = (_rel(gf[k], gd[k]), _rel(ge[k], gd[k]))
    return res


CASES = {
    'b4_128_b5_ref_train': dict(B=4, H=128, depths=SO.B5_DEPTHS, out=512, seed=10),
    'b32_128_b5_ref_train': dict(B=32, H=128, depths=SO.B5_DEPTHS, out=512, seed=20),
    'b4_128_b5_default_eval': dict(B=4, H=128, depths=SO.B5_DEPTHS, out=512, seed=30, init='default', train=False),
    'b3_160_2242': dict(B=3, H=160, depths=(2, 2, 4, 2), out=512, seed=40),
    'b2_256_1111': dict(B=2, H=256, depths=(1, 1, 1, 1), out=512, seed=50),
    'b2_32_1111': dict(B=2, H=32, depths=(1, 1, 1, 1), out=512, seed=55),   # stage 4 at 1 x 1, one key
    'b4_128_b5_stressed': dict(B=4, H=128, depths=SO.B5_DEPTHS, out=512, seed=60, stress=True),
}


@pytest.mark.parametrize('case', list(CASES))
def test_fused_matches_float64(case):
    res = _case(**CASES[case])
    worst = max(((k, v) for k, v in res.items() if k != 'features'), key=lambda kv: kv[1][0])
    print('\n%s: features %.2e (eager %.2e); worst gradient group %s %.2e (eager %.2e)'
          % (case, res['features'][0], res['features'][1], worst[0], worst[1][0], worst[1][1]))
    for k, (f, e) in sorted(res.items()):
        print('  %-40s fused %.2e  eager %.2e' % (k, f, e))
    assert res['features'][0] <= FEATURE_BAR, res['features']
    bad = {k: v for k, v in res.items() if k != 'features' and not v[0] <= GRAD_BAR}
    assert not bad, bad


def _fresh(depths=(1, 2, 2, 1), out=64, B=4, H=64, seed=70, train=True):
    p = SO.make_params(depths, out, seed, dtype=torch.float32)
    m = FS.enable_fused_segformer(load(make_segformer(out, depths), p).to(DEV).train(train))
    x = torch.randn(B, 3, H, H, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
    return m, x


def test_drop_path_masks_and_generator_state_match_the_eager_module():
    m, x = _fresh(depths=(2, 2, 3, 2))
    torch.manual_seed(80)
    want = FS.drop_scales(m, x.shape[0], DEV)
    state_eager = torch.cuda.get_rng_state()
    torch.manual_seed(80)
    with torch.no_grad():
        feats = m(x)
    assert torch.equal(torch.cuda.get_rng_state(), state_eager)
    # the module's own eager forward from the same seed: each drop_path call returns x * r with its
    # draw r, which must be exactly the scale the kernels were given
    FS.enable_fused_segformer(m, enabled=False)
    calls = []
    hooks = [blk.drop_path.register_forward_hook(lambda mod, i, o: calls.append((i[0], o)))
             for i in range(4) for blk in getattr(m, 'block%d' % (i + 1))]
    torch.manual_seed(80)
    with torch.no_grad():
        m(x)
    for h in hooks:
        h.remove()
    assert torch.equal(torch.cuda.get_rng_state(), state_eager)
    assert want.shape == (18, 4) and torch.equal(want[:2], torch.ones(2, 4, device=DEV))
    assert len(calls) == 18
    for k, (inp, out) in enumerate(calls):
        assert torch.equal(out, inp * want[k].view(-1, 1, 1)), k
    assert torch.isfinite(feats).all()


def test_two_backwards_give_the_same_bits():
    m, x = _fresh(train=False)
    g = torch.randn(4, 64, 16, 16, generator=torch.Generator().manual_seed(81)).to(DEV)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        m(x).backward(g)
        grads.append([t.grad.clone() for t in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


def test_an_image_gives_the_same_bits_alone_and_in_a_batch():
    m, x = _fresh(B=32, H=128, train=False, depths=(1, 1, 2, 1))
    with torch.no_grad():
        batch = m(x)
        alone = m(x[5:6].contiguous())
    assert torch.equal(batch[5:6], alone)


def test_no_grad_keeps_no_workspace():
    m, x = _fresh()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.no_grad():
        feats = m(x)
    torch.cuda.synchronize()
    assert feats.grad_fn is None
    assert torch.cuda.memory_allocated() - before == feats.numel() * 4


def test_second_backward_is_refused():
    m, x = _fresh()
    feats = m(x)
    feats.sum().backward(retain_graph=True)
    with pytest.raises(_lib.NfiError, match='twice'):
        feats.sum().backward()


def test_double_backward_is_refused():
    m, x = _fresh()
    with pytest.raises(_lib.NfiError, match='create_graph'):
        torch.autograd.grad(m(x).sum(), list(m.parameters())[0], create_graph=True)


def test_adam_step_through_data_parallel_matches_float64():
    depths, out, B, H = (1, 2, 2, 1), 64, 4, 64
    p = SO.make_params(depths, out, 90, dtype=torch.float32)
    m = FS.enable_fused_segformer(load(make_segformer(out, depths), p).to(DEV).train())
    dp = torch.nn.DataParallel(m, device_ids=[0])
    x = torch.randn(B, 3, H, H, generator=torch.Generator().manual_seed(91)).to(DEV)
    target = torch.randn(B, out, H // 4, H // 4, generator=torch.Generator().manual_seed(92)).to(DEV)
    torch.manual_seed(93)
    scales = FS.drop_scales(m, B, DEV)
    state = torch.cuda.get_rng_state()
    pd = {k: v.double().to(DEV).requires_grad_() for k, v in p.items()}
    loss_d = torch.nn.functional.smooth_l1_loss(SO.forward(pd, depths, x.double(), list(scales.double())),
                                                target.double())
    loss_d.backward()
    opt = torch.optim.Adam(m.parameters(), lr=1e-4)
    torch.manual_seed(93)
    loss = torch.nn.functional.smooth_l1_loss(dp(x), target)
    opt.zero_grad()
    loss.backward()
    grads = {n: t.grad.clone() for n, t in m.named_parameters()}
    opt.step()
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert abs(loss.item() - loss_d.item()) <= 1e-4 * abs(loss_d.item())
    gf, gd = _groups(grads), _groups({n: t.grad for n, t in pd.items()})
    worst = max(_rel(gf[k], gd[k]) for k in gd)
    assert worst <= GRAD_BAR, worst


def _coord_loss(out, target_coords, target_mask, target_w):
    """train_coord_regressor's loss (run.py:1648-1663)."""
    pred_coords, pred_mask, pred_w = out
    loss_coords = (pred_coords - target_coords).norm(dim=-1).mul(target_mask).mean()
    return loss_coords + torch.nn.L1Loss()(pred_mask, target_mask) + torch.nn.MSELoss()(pred_w, target_w)


def test_encoder_step_through_both_opt_ins_matches_float64():
    """One train_coord_regressor step on the reference BootstrapEncoder with the fused backbone and
    the fused heads (nn.DataParallel on one device, drop path on, criteria, loss.backward(),
    Adam.step()) against the float64 module run with the same masks, on the heads' ReLU branches;
    and the CUDA generator's state after the step against the eager arm's."""
    from nerf_from_image_b200.encoder import enable_fused_encoder, saved_activations
    from oracle import encoder_oracle as EO
    from tests.encoder_standin import reference_encoder
    B, R, LAT, SEED = 4, 128, 64, 23
    torch.manual_seed(21)
    base = reference_encoder(LAT)
    if base is None:
        pytest.skip('needs the installed reference BootstrapEncoder')
    state = {k: v.clone() for k, v in base.state_dict().items()}
    g = torch.Generator().manual_seed(22)
    img = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).to(DEV)
    tgt = (torch.randn(B, R, R, 3, generator=g).to(DEV), (torch.rand(B, R, R, generator=g) > 0.5).float().to(DEV),
           torch.randn(B, 1, LAT, generator=g).to(DEV))
    runs, rng = {}, {}
    for name in ('fused', 'eager'):
        m = reference_encoder(LAT)
        m.load_state_dict(state)
        if name == 'fused':
            enable_fused_encoder(m)
            FS.enable_fused_segformer(m.backbone)
        m = m.to(DEV).train()
        model = torch.nn.DataParallel(m, [0])
        opt = torch.optim.Adam(model.parameters(), lr=6e-5)
        if name == 'fused':
            torch.manual_seed(SEED)
            scales = FS.drop_scales(m.backbone, B, DEV)
        torch.manual_seed(SEED)
        opt.zero_grad()
        out = model(img)
        if name == 'fused':
            branches = EO.branches_from_saved(saved_activations(out[0]))
        loss = _coord_loss(out, *tgt)
        loss.backward()
        runs[name] = (loss.item(), {k: v.grad.detach().clone() for k, v in m.named_parameters()})
        opt.step()
        rng[name] = torch.cuda.get_rng_state()
        assert all(torch.isfinite(p).all() for p in m.parameters())
    assert torch.equal(rng['fused'], rng['eager'])
    # float64: the backbone on the oracle with the fused arm's masks, the heads on its branches
    m = reference_encoder(LAT)
    m.load_state_dict(state)
    m = m.to(DEV, torch.float64).train()
    feats = SO.forward(dict(m.backbone.named_parameters()), SO.B5_DEPTHS, img.double(), list(scales.double()))
    maps, pooled = EO.heads(EO.params_of(m), feats, feats, branches)
    out = (maps[:, :3].permute(0, 2, 3, 1), torch.sigmoid(maps[:, 3]), m.w_regressor_post(pooled).unsqueeze(1))
    loss_d = _coord_loss(out, *[t.double() for t in tgt])
    loss_d.backward()
    ref = {k: v.grad for k, v in m.named_parameters()}
    rel_loss = {n: abs(runs[n][0] - loss_d.item()) / abs(loss_d.item()) for n in runs}
    print('\nencoder step vs float64: loss fused %.2e, eager fp32 %.2e' % (rel_loss['fused'], rel_loss['eager']))
    assert rel_loss['fused'] < 1e-4
    groups = {}
    for k in ref:
        key = k if k.startswith(('post', 'w_regressor_pre')) else k.split('.')[0]
        if k.startswith('backbone.'):
            key = 'backbone.' + _group(k[len('backbone.'):])
        groups.setdefault(key, []).append(k)
    worst = {}
    for grp, ks in groups.items():
        cat = lambda gs: torch.cat([gs[k].double().flatten() for k in ks])
        worst[grp] = (_rel(cat(runs['fused'][1]), cat(ref)), _rel(cat(runs['eager'][1]), cat(ref)))
    top = max(worst.items(), key=lambda kv: kv[1][0])
    print('  worst gradient group %s: fused %.2e, eager fp32 %.2e (%d groups)' % (top[0], *top[1], len(worst)))
    for grp in sorted(worst):
        if not grp.startswith('backbone.'):
            print('  %-24s fused %.2e, eager fp32 %.2e' % (grp, *worst[grp]))
    bad = {k: v for k, v in worst.items() if not v[0] < GRAD_BAR}
    assert not bad, bad


def test_a_refused_call_draws_no_masks():
    m, x = _fresh()
    m.double()   # fp64 parameters are outside the envelope
    state = torch.cuda.get_rng_state()
    with pytest.raises(_lib.NfiError, match='fp32'):
        m(x)
    assert torch.equal(torch.cuda.get_rng_state(), state)
