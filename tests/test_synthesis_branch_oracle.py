"""The float64 synthesis network on chosen leaky-ReLU branches (tests/synthesis_branch_oracle.py),
without a GPU:

1. on the masks of its own branches it is the plain oracle, bit for bit: planes, ws.grad, every
   parameter gradient and the double backward of ws.grad;
2. the mechanism behind the fused backward's float64 comparison: on a (64, 64, 64) net at 16^2
   (parameter seed 2) plain fp32 autograd through the oracle is 1.2e-3 from float64 because one
   pre-activation, 5.5e-8 from zero, takes the other branch; float64 on fp32's branches is 4e-7
   from fp32;
3. ``borrow_branches`` on fp32's pre-activations as the kernel's: it borrows exactly that one
   position, and refuses a forward error above its bound at a single position."""
import pytest
import torch

from fixtures import synthetic
from oracle import synthesis_oracle as SO
from tests import helpers_synth as HS
from tests import synthesis_branch_oracle as BO


def _double(p, grad=False):
    return {k: (v.double().requires_grad_(grad) if torch.is_tensor(v) and v.is_floating_point() else v)
            for k, v in p.items()}


def _case(seed, channels=(64, 64, 64), batch=3):
    """The net of the mechanism (parameter seed ``seed``; ws and g_planes drawn as the GPU tests
    draw them, Generator seed 8)."""
    res = 4 << (len(channels) - 1)
    p = synthetic.make_synthesis_params(seed, res, channels, 512)
    g = torch.Generator().manual_seed(8)
    ws = torch.randn(batch, 2 * len(channels), 512, generator=g)
    g_planes = torch.randn(batch, 3, res, res, 32, generator=g)
    g_img = g_planes.permute(0, 1, 4, 2, 3).reshape(batch, 96, res, res)
    return p, ws, g_img


def _grads(forward, p, ws, noises, g_img):
    """(img, ws.grad, parameter grads, HVP ws.grad) of L = <g_img, img> in float64."""
    pd = _double(p, grad=True)
    wd = ws.double().requires_grad_()
    nz = {k: v.double() for k, v in noises.items()}
    img = forward(pd, wd, nz)
    (gw,) = torch.autograd.grad(img, wd, g_img.double(), create_graph=True)
    t = torch.randn(ws.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    (hvp,) = torch.autograd.grad((gw * t).sum(), wd, retain_graph=True)
    keys = [k for k, v in pd.items() if torch.is_tensor(v) and v.requires_grad]
    pg = torch.autograd.grad(img, [pd[k] for k in keys], g_img.double(), allow_unused=True)
    return img.detach(), gw.detach(), dict(zip(keys, pg)), hvp


def test_own_branches_are_the_plain_oracle_bit_for_bit():
    p, ws, g_img = _case(2)
    noises = HS.const_noises(p)
    assert noises, 'the seeded net has noise on every layer'
    u64 = BO.preactivations(_double(p), ws.double(), {k: v.double() for k, v in noises.items()})
    assert len(u64) == len(BO.layer_names(p)) == 5
    masks = [u > 0 for u in u64]
    plain = _grads(SO.synthesis_forward, p, ws, noises, g_img)
    masked = _grads(lambda pd, wd, nz: BO.synthesis_forward(pd, wd, nz, masks)[0], p, ws, noises, g_img)
    for a, b in zip(plain[:2], masked[:2]):
        assert torch.equal(a, b)
    assert plain[2].keys() == masked[2].keys()
    for k in plain[2]:
        a, b = plain[2][k], masked[2][k]
        assert (a is None) == (b is None), k
        assert a is None or torch.equal(a, b), k
    assert torch.equal(plain[3], masked[3])


def _mechanism(seed):
    p, ws, g_img = _case(seed)
    noises = HS.const_noises(p)
    pd, nz = _double(p), {k: v.double() for k, v in noises.items()}
    w32 = ws.clone().requires_grad_()
    img32, u32 = BO.synthesis_forward(p, w32, noises)
    g32 = torch.autograd.grad(img32, w32, g_img)[0].double()
    u64 = BO.preactivations(pd, ws.double(), nz)
    want = BO.ws_grad(pd, ws.double(), nz, g_img.double())
    want_br = BO.ws_grad(pd, ws.double(), nz, g_img.double(), [u > 0 for u in u32])
    flips = [((a > 0) != (b > 0)) for a, b in zip(u32, u64)]
    return p, g32, want, want_br, u32, u64, flips


def test_one_branch_flip_moves_fp32_ws_grad_by_1e_3():
    p, g32, want, want_br, u32, u64, flips = _mechanism(2)
    e_plain, e_br = BO.max_rel(g32, want), BO.max_rel(g32, want_br)
    n = [int(f.sum()) for f in flips]
    at = [u[f].abs().max().item() for u, f in zip(u64, flips) if f.any()]
    print('seed 2: fp32 vs float64 %.2e, vs float64 on fp32 branches %.2e; flips per layer %s, '
          '|u64| there %s' % (e_plain, e_br, n, ['%.1e' % a for a in at]))
    assert e_plain > 5e-4
    assert e_br < 2e-6
    assert sum(n) == 1 and n[BO.layer_names(p).index('b16.conv1')] == 1
    assert at[0] < 1e-6
    # the rows carry it up to and including b16.conv1's, not the last ToRGB row
    row = ((g32 - want).norm(dim=(0, 2)) / want.norm(dim=(0, 2))).tolist()
    print('  per row %s' % ' '.join('%.1e' % r for r in row))
    assert row[-1] < 1e-5 and max(row[:-1]) > 1e-4


@pytest.mark.parametrize('seed', [1, 5])
def test_without_a_flip_fp32_is_at_rounding(seed):
    _, g32, want, want_br, _, _, flips = _mechanism(seed)
    assert not any(f.any() for f in flips)
    assert torch.equal(want, want_br)
    assert BO.max_rel(g32, want) < 2e-6, BO.max_rel(g32, want)


def test_borrow_branches_guard():
    p, _, _, _, u32, u64, _ = _mechanism(2)
    u_cl = [u.detach().permute(0, 2, 3, 1) for u in u32]
    masks, borrowed = BO.borrow_branches(p, u_cl, u64, 4e-5)   # fp32's u: 2.5e-6 off
    assert borrowed == {'b4.conv1': 0, 'b8.conv0': 0, 'b8.conv1': 0, 'b16.conv0': 0, 'b16.conv1': 1}
    assert all(torch.equal(m, u > 0) for m, u in zip(masks, u32))
    # one position of one layer off by more than tau / 4: refused
    u_bad = [u.clone() for u in u_cl]
    u_bad[2][0, 3, 5, 7] += 2e-5
    with pytest.raises(AssertionError, match='forward u error'):
        BO.borrow_branches(p, u_bad, u64, 4e-5)
