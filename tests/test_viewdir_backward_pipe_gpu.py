"""--use_viewdir inversion backward on the pipelined tensor-core kernel (render_backward_pipe<...,
VD = true>, csrc/nfi_pipe_vd.cu): decoder and mapper output frozen; gradients to the planes,
palette, beta / alpha, the camera and the per-ray view features.

Mode 4 (NFI_MLP_TC_PIPE) and mode 1 (the fp32 SIMT view kernel) meet the same float64 bars, and
their view-feature gradients differ in the last bits, so a silent SIMT route is caught.  Requests
outside the kernel's envelope (decoder / W3 / b3 gradients, a small workspace) give the SIMT
kernel's results bit for bit.
"""
import math

import pytest
import torch

from fixtures import synthetic
from nerf_from_image_b200 import _lib
from nerf_from_image_b200.fused import RenderConfig, fused_render
from tests import helpers as Hh

pytestmark = pytest.mark.gpu

H, W, S = 24, 40, 16
TC, SIMT = 4, 1
FIELD = ('planes', 'palette', 'beta', 'alpha')
CAMERA = ('c2w', 'focal', 'center', 'bbox')


def make(case, A=10, batch=2, seed=3):
    scene, cams = Hh.make_case(case, seed=seed, batch=batch, plane_res=32, attention_values=A)
    return synthetic.add_view_mapper(scene), cams


def dbl(d):
    return {k: (v.double() if torch.is_tensor(v) else v) for k, v in d.items()}


def weights(B, h, w, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, h, w, 3, generator=g), torch.randn(B, h, w, generator=g),
            torch.randn(B, h, w, 3, generator=g))


def oracle_grads(scene, cams, nt, nu, vf, h, w, kw, coords=False):
    """float64 autograd of sum(rgb wr) + sum(mask wm) (+ sum(coords we))."""
    sc, cm = dbl(scene), dbl(cams)
    names = [n for n in FIELD if sc.get(n) is not None] + [n for n in CAMERA if cm.get(n) is not None]
    for n in names:
        d = sc if n in FIELD else cm
        d[n] = d[n].clone().requires_grad_()
    vfl = vf.double().clone().requires_grad_()
    out = Hh.run_oracle(sc, cm, h, w, S, nt.double() if nt is not None else None,
                        nu.double() if nu is not None else None, view_features=vfl,
                        w3=sc['w3'], b3=sc['b3'], compute_coords=coords, **kw)
    wr, wm, we = (x.to(out['rgb'].device).double() for x in weights(vf.shape[0], h, w))
    loss = (out['rgb'] * wr).sum() + (out['mask'] * wm).sum()
    if coords:
        loss = loss + (out['semantics'] * we).sum()
    lv = [sc[n] if n in FIELD else cm[n] for n in names] + [vfl]
    gr = torch.autograd.grad(loss, lv, allow_unused=True)
    return {n: x for n, x in zip(names + ['view_features'], gr) if x is not None}


def cuda_grads(scene, cams, nt, nu, vf, h, w, kw, mode, coords=False, cam_grad=True,
               vf_grad=True, decoder_grad=(), rows=None, wts=None):
    sc, cm = Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda')
    names = [n for n in FIELD if sc.get(n) is not None]
    if cam_grad:
        names += [n for n in CAMERA if cm.get(n) is not None]
    names += list(decoder_grad)
    for n in names:
        d = cm if n in CAMERA else sc
        d[n] = d[n].clone().requires_grad_()
    vfl = vf.cuda().clone().requires_grad_(vf_grad)
    cfg = RenderConfig(scene_range=sc['scene_range'], white_background=sc['white_background'],
                       use_sdf=kw.get('use_sdf', True), fine_sampling=kw.get('fine_sampling', True),
                       attention_values=sc['palette'].shape[1] if sc['palette'] is not None else 0,
                       mlp_mode=mode)
    rgb, _, mask, extra = fused_render(
        sc['planes'], sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'], sc['beta'],
        sc['alpha'], cm['c2w'], cm['focal'], cm['center'], cm['bbox'], cfg, h, w, S,
        nt.cuda() if nt is not None else None, nu.cuda() if nu is not None else None,
        _lib.EXTRA_COORDS if coords else _lib.EXTRA_NONE, cam_grad,
        view=(vfl, sc['w3'], sc['b3']), rows=rows)
    wr, wm, we = (x.cuda() for x in (wts or weights(vf.shape[0], h, w)))
    loss = (rgb * wr).sum() + (mask * wm).sum()
    if coords:
        loss = loss + (extra * we).sum()
    lv = [sc[n] if n in FIELD or n in decoder_grad else cm[n] for n in names]
    lv += [vfl] if vf_grad else []
    gr = torch.autograd.grad(loss, lv, allow_unused=True)
    out = {n: x for n, x in zip(names + (['view_features'] if vf_grad else []), gr) if x is not None}
    return out, (rgb, mask)


def check(have, want, label):
    errs = {}
    for n, b in want.items():
        a = have[n].detach().double().to(b.device)
        errs[n] = Hh.rel_l2(a, b)
        tol = 5e-3 if n in ('beta', 'alpha') else 1e-3
        assert errs[n] < tol, (label, n, errs[n])
    print('\n  %s: ' % label + ', '.join('%s %.1e' % kv for kv in errs.items()))


def inputs(case, A, h, w, batch=2, randomize=True, seed=3):
    scene, cams = make(case, A, batch, seed)
    nt, nu = synthetic.make_noise(7, batch, h, w, S) if randomize else (None, None)
    vf = Hh.view_features(scene, cams, h, w).detach()
    return scene, cams, nt, nu, vf


@pytest.mark.parametrize('case,A,kw', [
    ('p3d_bbox', 10, {}),
    ('cub_ortho', 10, {}),
    ('chairs_white_center', 0, {}),
    ('p3d_plain', 15, {}),
    ('p3d_plain', 10, dict(coords=True)),
    ('p3d_plain', 10, dict(fine_sampling=False)),
    ('p3d_plain', 10, dict(use_sdf=False)),
    ('p3d_plain', 10, dict(randomize=False)),
])
def test_inversion_gradients_match_float64_on_both_kernels(cuda_lib, case, A, kw):
    kw = dict(kw)
    coords, randomize = kw.pop('coords', False), kw.pop('randomize', True)
    scene, cams, nt, nu, vf = inputs(case, A, H, W, randomize=randomize)
    want = oracle_grads(scene, cams, nt, nu, vf, H, W, kw, coords)
    tc, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, kw, TC, coords)
    simt, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, kw, SIMT, coords)
    assert set(tc) == set(want) == set(simt)
    check(tc, want, 'tensor core')
    check(simt, want, 'SIMT')
    # the two kernels sum in different orders: equal results would mean one kernel ran twice
    assert not torch.equal(tc['view_features'], simt['view_features'])


def test_multiwave_batch_against_float64_and_per_image_bit_exact(cuda_lib):
    """A ragged batch with more than two waves of tiles per CTA: the look-ahead fwd(m + 1) crosses
    tile boundaries, and each ray's view-feature gradient (written once, without atomics) equals
    the same ray's of its image rendered alone, bit for bit."""
    B, h, w = 4, 100, 90
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_tiles = B * math.ceil(h / 8) * math.ceil(w / 16)
    assert n_tiles > 2 * sms, (n_tiles, sms)
    scene, cams, nt, nu, vf = inputs('p3d_plain', 10, h, w, batch=B, seed=5)
    full, _ = cuda_grads(scene, cams, nt, nu, vf, h, w, {}, TC)
    want = oracle_grads(Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda'), nt.cuda(),
                        nu.cuda(), vf.cuda(), h, w, {})
    check(full, want, 'batch of %d tiles' % n_tiles)
    for b in range(B):
        sc = {k: (v[b:b + 1] if k in ('planes', 'palette') and v is not None else v)
              for k, v in scene.items()}
        cm = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cams.items()}
        nu_b = nu.view(B, h * w, S)[b].contiguous()
        alone, _ = cuda_grads(sc, cm, nt[b:b + 1], nu_b, vf[b:b + 1], h, w, {}, TC,
                              wts=[x[b:b + 1] for x in weights(B, h, w)])
        assert torch.equal(alone['view_features'][0], full['view_features'][b]), b


def test_edge_rays_and_row_band(cuda_lib):
    """33 x 21: padding rows of the edge tiles carry the clamped edge ray's view features but must
    not overwrite its gradient; a band of rows gives the same rows' gradients bit for bit."""
    h, w, r0 = 21, 33, 8
    scene, cams, nt, nu, vf = inputs('p3d_plain', 10, h, w)
    want = oracle_grads(scene, cams, nt, nu, vf, h, w, {})
    have, _ = cuda_grads(scene, cams, nt, nu, vf, h, w, {}, TC)
    check(have, want, '21 x 33')
    gv, wv = have['view_features'].cpu().double(), want['view_features']
    for name, a, b in (('last column', gv[:, :, -1], wv[:, :, -1]),
                       ('last row', gv[:, -1], wv[:, -1])):
        assert b.abs().max() > 0
        assert Hh.rel_l2(a, b) < 1e-3, (name, Hh.rel_l2(a, b))
    from nerf_from_image_b200 import parallel as PAR
    nt_r, nu_r = PAR.slice_rows(nt, nu, 2, h, w, r0, h)
    band, _ = cuda_grads(scene, cams, nt_r, nu_r, vf[:, r0:].contiguous(), h - r0, w, {}, TC,
                         cam_grad=False, rows=(r0, h), wts=[x[:, r0:] for x in weights(2, h, w)])
    full, _ = cuda_grads(scene, cams, nt, nu, vf, h, w, {}, TC, cam_grad=False)
    assert torch.equal(band['view_features'], full['view_features'][:, r0:])


def test_zero_output_layer(cuda_lib):
    scene, cams, nt, nu, vf = inputs('p3d_plain', 10, H, W)
    scene = dict(scene, w3=torch.zeros_like(scene['w3']), b3=torch.zeros_like(scene['b3']))
    want = oracle_grads(scene, cams, nt, nu, vf, H, W, {})
    have, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC)
    assert torch.count_nonzero(have['view_features']).item() == 0
    assert Hh.rel_l2(have['planes'].cpu().double(), want['planes']) < 1e-3


def test_without_camera_gradient(cuda_lib):
    """cam_grad=False with detached view features (force_no_cam_grad): grad_view_features is
    NULL in the kernel; the plane gradient is still right."""
    scene, cams, nt, nu, vf = inputs('p3d_bbox', 10, H, W)
    want = oracle_grads(scene, cams, nt, nu, vf, H, W, {})
    have, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC, cam_grad=False, vf_grad=False)
    assert set(have) == {'planes', 'palette', 'beta', 'alpha'}
    for n in have:
        assert Hh.rel_l2(have[n].cpu().double(), want[n]) < (5e-3 if n in ('beta', 'alpha') else 1e-3)


def test_requests_outside_the_envelope_take_the_simt_kernel(cuda_lib, monkeypatch):
    """Decoder or W3 / b3 gradients (the GAN step), or a workspace below
    NFI_VIEW_BACKWARD_WORKSPACE_BYTES: the SIMT view kernel, whose per-ray outputs (written without
    atomics) are deterministic -- and differ in the last bits from the tensor-core kernel's."""
    scene, cams, nt, nu, vf = inputs('p3d_plain', 10, H, W)
    tc, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC)
    dec, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC, decoder_grad=('w1',))
    head, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC, decoder_grad=('w3', 'b3'))
    monkeypatch.setattr(_lib, 'VIEW_BACKWARD_WORKSPACE_BYTES', _lib.VIEW_BACKWARD_WORKSPACE_BYTES - 256)
    small, _ = cuda_grads(scene, cams, nt, nu, vf, H, W, {}, TC)
    for other in (dec, head):
        assert torch.equal(other['view_features'], small['view_features'])
        assert torch.equal(other['c2w'], small['c2w'])
    assert not torch.equal(tc['view_features'], small['view_features'])
