"""The bootstrap encoder's fused heads (include/nfi_encoder.h) on the GPU against float64.

Every comparison is rel-L2 against float64 on the GPU.  On the kernel's own ReLU branches (read from
the saved activations) the outputs are held to 1e-4 and every gradient group to 3e-4, after checking
that wherever the kernel and float64 disagree on a branch the float64 pre-activation is below 1e-3
of its layer's RMS.  The plain float64 figures (float64 taking its own branches) and the eager fp32
module's (TF32 off) are printed beside them."""
import pytest
import torch
from torch import nn

from nerf_from_image_b200 import _lib
from nerf_from_image_b200.encoder import enable_fused_encoder, heads, saved_activations
from oracle import encoder_oracle as EO
from tests.encoder_standin import StandInBootstrapEncoder, load_params, reference_encoder

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a GPU')]

DEV = 'cuda:0'
OUT_BAR, GRAD_BAR = 1e-4, 3e-4


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _case(B, h, w, seed, pose=True, latent=True, separate=False):
    """A module with seeded heads on the GPU, and seeded features / output gradients."""
    enc = StandInBootstrapEncoder(64, pose_regressor=pose, latent_regressor=latent,
                                  separate_backbones=separate)
    p = EO.make_params(seed=seed)
    load_params(enc, p)
    enc = enc.to(DEV).train()
    g = torch.Generator().manual_seed(seed + 1)
    f = torch.randn(B, 512, h, w, generator=g).to(DEV) if pose or not separate else None
    fl = (torch.randn(B, 512, h, w, generator=g).to(DEV) if separate else f) if latent else None
    if not pose:
        f = None
    gm = torch.randn(B, 4 * h, 4 * w, 4, generator=g).to(DEV) if pose else None
    gp = torch.randn(B, 512, generator=g).to(DEV) if latent else None
    return enc, f, fl, gm, gp


def _leaves(f, fl):
    a = f.clone().requires_grad_() if f is not None else None
    b = (a if fl is f else fl.clone().requires_grad_()) if fl is not None else None
    return a, b


def _fused(enc, f, fl, gm, gp, keep_saved=True):
    a, b = _leaves(f, fl)
    maps, pooled = heads(enc, a, b)
    saved = saved_activations(maps if gm is not None else pooled) if keep_saved else None
    loss = 0
    if gm is not None:
        loss = loss + (maps * gm).sum()
    if gp is not None:
        loss = loss + (pooled * gp).sum()
    loss.backward()
    grads = {'features': a.grad if a is not None else None}
    if b is not None and b is not a:
        grads['features_latent'] = b.grad
    for k, t in EO.params_of(enc).items():
        grads[k] = t.grad.clone()
        t.grad = None
    return maps.detach(), pooled.detach(), grads, saved


def _reference(enc, f, fl, gm, gp, dtype, branches=None):
    p = {k: v.detach().to(dtype).requires_grad_() for k, v in EO.params_of(enc).items()}
    a = f.to(dtype).clone().requires_grad_() if f is not None else None
    b = None if fl is None else (a if fl is f else fl.to(dtype).clone().requires_grad_())
    maps, pooled = EO.heads(p, a, b, branches)
    loss = 0
    if maps is not None:
        maps = maps.permute(0, 2, 3, 1)
        loss = loss + (maps * gm.to(dtype)).sum()
    if pooled is not None:
        loss = loss + (pooled * gp.to(dtype)).sum()
    loss.backward()
    grads = {'features': a.grad if a is not None else None}
    if b is not None and b is not a:
        grads['features_latent'] = b.grad
    grads.update({k: t.grad for k, t in p.items()})
    return maps, pooled, grads, p, a, b


def _check_branches(enc, f, fl, saved):
    """Where the kernel's branch differs from float64's (given the kernel's upstream branches), the
    float64 pre-activation is within 1e-3 of its layer's RMS of zero."""
    br = EO.branches_from_saved(saved)
    p = {k: v.detach().double() for k, v in EO.params_of(enc).items()}
    u = EO.pre_activations(p, f.double() if f is not None else None,
                           fl.double() if fl is not None else None, br)
    flips = {}
    for k, v in u.items():
        bad = (v > 0) != br[k]
        rms = v.square().mean().sqrt()
        if bad.any():
            assert v[bad].abs().max() < 1e-3 * rms, (k, v[bad].abs().max().item(), rms.item())
        flips[k] = int(bad.sum())
    return br, flips


def _compare(B, h, w, seed, label, **kw):
    enc, f, fl, gm, gp = _case(B, h, w, seed, **kw)
    maps, pooled, grads, saved = _fused(enc, f, fl, gm, gp)
    br, flips = _check_branches(enc, f, fl, saved)
    m64, p64, g64 = _reference(enc, f, fl, gm, gp, torch.float64, br)[:3]
    mp, pp, gplain = _reference(enc, f, fl, gm, gp, torch.float64)[:3]
    m32, p32, g32 = _reference(enc, f, fl, gm, gp, torch.float32)[:3]
    errs = {}
    if m64 is not None:
        errs['coords'] = (_rel(maps[..., :3], m64[..., :3]), _rel(maps[..., :3], mp[..., :3]),
                          _rel(m32[..., :3], mp[..., :3]))
        errs['mask logit'] = (_rel(maps[..., 3], m64[..., 3]), _rel(maps[..., 3], mp[..., 3]),
                              _rel(m32[..., 3], mp[..., 3]))
    if p64 is not None:
        errs['pooled'] = (_rel(pooled, p64), _rel(pooled, pp), _rel(p32, pp))
    for k in g64:
        if g64[k] is not None:
            errs[k] = (_rel(grads[k], g64[k]), _rel(grads[k], gplain[k]), _rel(g32[k], gplain[k]))
    print('\n%s: branch flips %s' % (label, flips))
    for k, (e_br, e_plain, e_eager) in errs.items():
        print('  %-16s rel-L2 vs float64: on branches %.2e, plain %.2e; eager fp32 %.2e'
              % (k, e_br, e_plain, e_eager))
    for k, (e_br, _, _) in errs.items():
        bar = OUT_BAR if k in ('coords', 'mask logit', 'pooled') else GRAD_BAR
        assert e_br < bar, (label, k, e_br)
    return errs


def test_heads_at_training_shape(cuda_lib):
    _compare(4, 32, 32, seed=11, label='B=4 128^2')


def test_heads_with_more_tiles_than_sms(cuda_lib):
    _compare(32, 32, 32, seed=12, label='B=32 128^2')


def test_heads_non_square(cuda_lib):
    _compare(3, 24, 40, seed=13, label='B=3 96x160')


@pytest.mark.parametrize('kw', [{'latent': False}, {'pose': False}, {'separate': True}],
                         ids=['pose_only', 'latent_only', 'separate'])
def test_head_combinations(cuda_lib, kw):
    _compare(4, 32, 32, seed=14, label=str(kw), **kw)


def test_backward_is_bit_identical_and_forward_batch_independent(cuda_lib):
    enc, f, fl, gm, gp = _case(32, 32, 32, seed=15)
    r1 = _fused(enc, f, fl, gm, gp, keep_saved=False)
    r2 = _fused(enc, f, fl, gm, gp, keep_saved=False)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1])
    for k in r1[2]:
        assert torch.equal(r1[2][k], r2[2][k]), k
    with torch.no_grad():
        k = 17
        one = heads(enc, f[k:k + 1].contiguous(), f[k:k + 1].contiguous())
        assert torch.equal(one[0][0], r1[0][k]) and torch.equal(one[1][0], r1[1][k])


def test_refusals(cuda_lib):
    enc, f, fl, gm, gp = _case(2, 8, 8, seed=16)
    with pytest.raises(_lib.NfiError):
        heads(enc, f.double(), f.double())                      # not fp32
    with pytest.raises(_lib.NfiError):
        heads(enc, f[:, :256].contiguous(), f[:, :256].contiguous())   # not 512 channels
    with pytest.raises(_lib.NfiError):
        heads(enc, torch.zeros(2, 512, 2000, 1, device=DEV), torch.zeros(2, 512, 2000, 1, device=DEV))
    a = f.clone().requires_grad_()
    maps, pooled = heads(enc, a, a)
    loss = maps.sum() + pooled.sum()
    loss.backward(retain_graph=True)
    with pytest.raises(_lib.NfiError):
        loss.backward()                                           # a second backward
    a = f.clone().requires_grad_()
    maps, pooled = heads(enc, a, a)
    with pytest.raises(_lib.NfiError):
        torch.autograd.grad(maps.sum() + pooled.sum(), a, create_graph=True)   # a double backward
    enc.eval()
    with pytest.raises(_lib.NfiError):
        heads(enc, f.clone().requires_grad_(), f)                 # gradient through eval mode
    with torch.no_grad():
        heads(enc, f, f)                                          # eval + no_grad: save = 0


def _coord_loss(out, target_coords, target_mask, target_w):
    """train_coord_regressor's loss (run.py:1648-1663)."""
    pred_coords, pred_mask, pred_w = out
    loss_coords = (pred_coords - target_coords).norm(dim=-1).mul(target_mask).mean()
    return loss_coords + nn.L1Loss()(pred_mask, target_mask) + nn.MSELoss()(pred_w, target_w)


def _float64_forward(m, x, branches):
    """The module's forward in float64 (the reference SegFormer casts its output to fp32: it is cast
    back), its heads on the oracle with the given ReLU branches (None: its own)."""
    features = m.backbone(x).double()
    maps, pooled = EO.heads(EO.params_of(m), features, features, branches)
    return (maps[:, :3].permute(0, 2, 3, 1), torch.sigmoid(maps[:, 3]),
            m.w_regressor_post(pooled).unsqueeze(1))


def test_training_step_through_the_drop_in(cuda_lib):
    """One train_coord_regressor step (forward, criteria, loss.backward(), Adam.step()) through
    nn.DataParallel on the fused module, against the float64 module on the kernel's branches."""
    B, R, LAT = 4, 128, 64
    build = lambda: (reference_encoder(LAT) or StandInBootstrapEncoder(LAT))
    torch.manual_seed(21)
    state = {k: v.clone() for k, v in build().state_dict().items()}
    g = torch.Generator().manual_seed(22)
    img = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).to(DEV)
    tgt = (torch.randn(B, R, R, 3, generator=g).to(DEV), (torch.rand(B, R, R, generator=g) > 0.5).float().to(DEV),
           torch.randn(B, 1, LAT, generator=g).to(DEV))
    runs, branches = {}, None
    for name in ('fused', 'eager', 'float64', 'float64 plain'):
        dtype = torch.float64 if name.startswith('float64') else torch.float32
        m = build()
        m.load_state_dict(state)
        if name == 'fused':
            enable_fused_encoder(m)
        m = m.to(DEV, dtype).train()
        m.backbone.eval()   # SegFormer's drop-path draws would differ between the arms
        model = nn.DataParallel(m, [0])
        model.requires_grad_(True)
        opt = torch.optim.Adam(model.parameters(), lr=6e-5)
        opt.zero_grad()
        x = img.to(dtype)
        if dtype == torch.float64:
            out = _float64_forward(m, x, branches if name == 'float64' else None)
        else:
            out = model(x)
        if name == 'fused':
            branches = EO.branches_from_saved(saved_activations(out[0]))
        loss = _coord_loss(out, *[t.to(dtype) for t in tgt])
        loss.backward()
        runs[name] = (loss.detach(), {k: v.grad.detach().clone() for k, v in m.named_parameters()})
        opt.step()
        assert all(torch.isfinite(p).all() for p in m.parameters())
    ref_loss, ref_g = runs['float64']
    rel_loss = lambda n: abs(runs[n][0].item() - ref_loss.item()) / abs(ref_loss.item())
    print('\ndrop-in step vs float64 on the kernel\'s branches: loss rel err fused %.2e, eager fp32 %.2e '
          '(plain float64 %.2e)' % (rel_loss('fused'), rel_loss('eager'), rel_loss('float64 plain')))
    assert rel_loss('fused') < OUT_BAR
    groups = {}
    for k in ref_g:
        groups.setdefault(k if k.startswith(('post', 'w_regressor_pre')) else k.split('.')[0], []).append(k)
    for grp, ks in groups.items():
        cat = lambda gs: torch.cat([gs[k].double().flatten() for k in ks])
        e = {n: _rel(cat(runs[n][1]), cat(ref_g)) for n in ('fused', 'eager', 'float64 plain')}
        print('  %-22s gradient rel-L2: fused %.2e, eager fp32 %.2e, plain float64 %.2e'
              % (grp, e['fused'], e['eager'], e['float64 plain']))
        assert e['fused'] < GRAD_BAR, (grp, e)
