"""--use_viewdir on the pipelined tensor-core forward kernel (render_forward_pipe<..., VD = true>,
csrc/nfi_pipe_vd.cu): layer 2 with N = 40, leaky ReLU of features + view features on the
accumulator registers, layer 3 on wgmma, all in 3xTF32.

Every test here names the kernel it wants (mlp_mode 4 = NFI_MLP_TC_PIPE refuses instead of falling
back; 1 = the fp32 SIMT view kernel, the control), so a silent fallback cannot pass.  The backward
of a view-conditioned render stays on render_backward_simt<..., VD>.
"""
import math

import pytest
import torch

from fixtures import synthetic
from nerf_from_image_b200 import _lib
from oracle import render_oracle as O
from tests import helpers as Hh

pytestmark = pytest.mark.gpu

H, W, S = 24, 40, 16
TC, SIMT, AUTO = 4, 1, 0


def make(case, A=10, batch=2, res=32, seed=3):
    scene, cams = Hh.make_case(case, seed=seed, batch=batch, plane_res=res, attention_values=A)
    return synthetic.add_view_mapper(scene), cams


def z_fine_of(out):
    fn = out[0].grad_fn
    return dict(zip(fn.saved_names, fn.saved_tensors))['z_fine']


def extra_mode_of(kw):
    return (_lib.EXTRA_COORDS if kw.get('compute_coords') else
            _lib.EXTRA_SEMANTICS if kw.get('compute_semantics') else _lib.EXTRA_NONE)


@pytest.mark.parametrize('case,A,kw', [
    ('p3d_bbox', 10, {}),
    ('cub_ortho', 10, {}),
    ('chairs_white_center', 0, {}),
    ('p3d_plain', 15, {}),
    ('p3d_plain', 10, dict(compute_semantics=True)),
    ('p3d_plain', 10, dict(compute_coords=True)),
    ('p3d_plain', 10, dict(fine_sampling=False)),
    ('p3d_plain', 10, dict(use_sdf=False)),
    ('p3d_plain', 10, dict(randomize=False)),
])
def test_forward_matches_oracle(cuda_lib, case, A, kw):
    scene, cams = make(case, A)
    kw = dict(kw)
    randomize = kw.pop('randomize', True)
    nt, nu = synthetic.make_noise(7, 2, H, W, S) if randomize else (None, None)
    want = Hh.run_oracle(scene, cams, H, W, S, nt, nu, **kw)
    extra_mode = extra_mode_of(kw)
    with torch.no_grad():
        rgb, depth, mask, extra = Hh.run_cuda(scene, cams, H, W, S, nt, nu,
                                              use_sdf=kw.get('use_sdf', True),
                                              fine_sampling=kw.get('fine_sampling', True),
                                              extra_mode=extra_mode, mlp_mode=TC)
    tol = 1e-3 if not randomize else 2e-4   # randomize=False: sample 0 sits on the cube face
    assert Hh.rel_l2(rgb.cpu(), want['rgb']) < tol
    assert Hh.rel_l2(mask.cpu(), want['mask']) < tol
    assert Hh.rel_l2(depth.cpu(), want['depth']) < tol
    if extra_mode:
        assert Hh.rel_l2(extra.cpu(), want['semantics']) < tol


def test_semantics_of_a_three_entry_palette_stay_on_the_simt_kernel(cuda_lib):
    """Outside the pipelined kernel's envelope: the explicit mode refuses, AUTO renders."""
    scene, cams = make('p3d_plain', 3)
    nt, nu = synthetic.make_noise(7, 2, H, W, S)
    want = Hh.run_oracle(scene, cams, H, W, S, nt, nu, compute_semantics=True)
    with torch.no_grad():
        with pytest.raises(_lib.NfiError):
            Hh.run_cuda(scene, cams, H, W, S, nt, nu, extra_mode=_lib.EXTRA_SEMANTICS, mlp_mode=TC)
        out = Hh.run_cuda(scene, cams, H, W, S, nt, nu, extra_mode=_lib.EXTRA_SEMANTICS,
                          mlp_mode=AUTO)
    assert Hh.rel_l2(out[0].cpu(), want['rgb']) < 2e-4
    assert Hh.rel_l2(out[3].cpu(), want['semantics']) < 2e-4


# Measured on an H100 (rgb, mask rel-L2; z_fine max-abs over the ray span): p3d_plain 24x40
# 6.0e-6, 5.9e-6, 4.7e-6; chairs A = 0 1.8e-6, 3.4e-6, 5.2e-6; cub_ortho 21x33 1.8e-5, 1.9e-5,
# 1.6e-5.  The orthographic case's fine depths get their own bar: the inverse CDF moves a sample
# by (CDF error) / pdf, and its rays cross long low-density bins -- the sensitivity
# tests/test_multiwave_gpu.py (Z_FINE_BARS) documents for the same dataset, where the oracle's own
# fp32 run sits 4.8e-5 from float64.
@pytest.mark.parametrize('case,A,h,w,z_bar', [('p3d_plain', 10, H, W, 1e-5),
                                              ('chairs_white_center', 0, H, W, 1e-5),
                                              ('p3d_plain', 10, 21, 33, 1e-5),
                                              ('cub_ortho', 15, 21, 33, 3e-5)])
def test_matches_the_simt_kernel_at_fp32_level(cuda_lib, case, A, h, w, z_bar):
    """3xTF32 through three layers against the fp32 FFMA kernel on the same inputs."""
    scene, cams = make(case, A)
    nt, nu = synthetic.make_noise(11, 2, h, w, S)
    sc = dict(scene, planes=scene['planes'].clone().requires_grad_())  # keeps z_fine readable
    a = Hh.run_cuda(sc, cams, h, w, S, nt, nu, mlp_mode=TC)
    b = Hh.run_cuda(sc, cams, h, w, S, nt, nu, mlp_mode=SIMT)
    o, d = O.ray_bundle(h, w, cams['focal'], cams['c2w'], cams['bbox'], cams['center'])
    near, far, hit = O.near_far_planes(o, torch.nn.functional.normalize(d, dim=-1),
                                       scene['scene_range'])[:3]
    span = (far - near).abs().reshape(-1)[hit.reshape(-1)].cuda()
    dz = (z_fine_of(a) - z_fine_of(b)).abs()[hit.reshape(-1).cuda()].max(dim=-1).values / span
    errs = dict(rgb=Hh.rel_l2(a[0].detach(), b[0].detach()),
                mask=Hh.rel_l2(a[2].detach(), b[2].detach()), z_fine=dz.max().item())
    print('\n  tensor-core vs SIMT: ' + ', '.join('%s %.2e' % kv for kv in errs.items()))
    assert errs['rgb'] < 2e-5 and errs['mask'] < 2e-5 and errs['z_fine'] < z_bar, errs


def carla_scene(B, res, A=10, seed=21, device='cuda'):
    """The CARLA dataset_config: scene_range 3.0, white background, perspective cameras."""
    scene = synthetic.make_scene(seed, B, plane_res=res, attention_values=A, scene_range=3.0,
                                 white_background=True, object_radius=1.5, device=device)
    cams = synthetic.make_cameras(seed, B, ortho=False, radius=6.4, device=device)
    return synthetic.add_view_mapper(scene), cams


def dbl(d):
    return {k: (v.double() if torch.is_tensor(v) else
                ({a: b.double() for a, b in v.items()} if isinstance(v, dict) else v))
            for k, v in d.items()}


def image(scene, cams, nt, nu, b, h, w):
    sc = {k: (v[b:b + 1] if k in ('planes', 'palette') and v is not None else v)
          for k, v in scene.items()}
    cm = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cams.items()}
    return sc, cm, nt[b:b + 1], nu.view(-1, h * w, nu.shape[-1])[b].contiguous()


def test_training_scale_over_several_waves(cuda_lib):
    """256^2 planes, 128 x 128 rays, 64 + 64 samples, 3 images = 768 tiles on the persistent grid
    (more than five per CTA on 132 SMs): each image against the float64 oracle, and each image
    rendered alone equal to its slice of the batch bit for bit -- neither the per-tile view
    features nor the persistent loop carry state across tiles."""
    B, h, w, s = 3, 128, 128, 64
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_tiles = B * math.ceil(h / 8) * math.ceil(w / 16)
    assert n_tiles >= 2 * sms, (n_tiles, sms)
    scene, cams = carla_scene(B, 256)
    nt, nu = synthetic.make_noise(31, B, h, w, s, device='cuda')
    with torch.no_grad():
        full = Hh.run_cuda(scene, cams, h, w, s, nt, nu, mlp_mode=TC)[:3]
        for b in range(B):
            sc, cm, nt_b, nu_b = image(scene, cams, nt, nu, b, h, w)
            alone = Hh.run_cuda(sc, cm, h, w, s, nt_b, nu_b, mlp_mode=TC)[:3]
            for n, x, y in zip(('rgb', 'depth', 'mask'), alone, full):
                assert torch.equal(x[0], y[b]), (b, n, (x[0] - y[b]).abs().max().item())
            ref = Hh.run_oracle(dbl(sc), dbl(cm), h, w, s, nt_b.double(), nu_b.double())
            err = Hh.rel_l2(full[0][b].double(), ref['rgb'][0])
            print('\n  image %d rgb rel-L2 vs float64 %.2e' % (b, err))
            assert err < 1e-4, (b, err)
            del ref


def test_a_row_band_equals_the_same_rows_of_the_full_image(cuda_lib):
    from nerf_from_image_b200 import parallel as PAR
    from nerf_from_image_b200.fused import RenderConfig, fused_render
    h, w, r0 = 21, 33, 8
    scene, cams = make('p3d_plain')
    sc, cm = Hh.to_device(scene, 'cuda'), Hh.to_device(cams, 'cuda')
    vm = {k: v.cuda() for k, v in scene['view_mapper'].items()}
    nt, nu = synthetic.make_noise(17, 2, h, w, S, device='cuda')
    vf = Hh.view_features(dict(sc, view_mapper=vm), cm, h, w)
    cfg = RenderConfig(scene_range=sc['scene_range'], white_background=sc['white_background'],
                       attention_values=10, mlp_mode=TC)

    def render(rows, hh, nt_, nu_, vf_):
        with torch.no_grad():
            return fused_render(sc['planes'], sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                                sc['beta'], sc['alpha'], cm['c2w'], cm['focal'], cm['center'],
                                cm['bbox'], cfg, hh, w, S, nt_, nu_, rows=rows,
                                view=(vf_, sc['w3'], sc['b3']))[:3]
    full = render(None, h, nt, nu, vf)
    nt_r, nu_r = PAR.slice_rows(nt, nu, 2, h, w, r0, h)
    band = render((r0, h), h - r0, nt_r, nu_r, vf[:, r0:].contiguous())
    for n, x, y in zip(('rgb', 'depth', 'mask'), band, full):
        assert torch.equal(x, y[:, r0:]), (n, (x - y[:, r0:]).abs().max().item())


def test_the_view_direction_matters(cuda_lib):
    scene, cams = make('p3d_plain')
    nt, nu = synthetic.make_noise(7, 2, H, W, S)
    with torch.no_grad():
        a = Hh.run_cuda(scene, cams, H, W, S, nt, nu, mlp_mode=TC)[0]
        flat = dict(scene, view_mapper={k: torch.zeros_like(v) for k, v in scene['view_mapper'].items()})
        b = Hh.run_cuda(flat, cams, H, W, S, nt, nu, mlp_mode=TC)[0]
    assert Hh.rel_l2(a, b) > 1e-2


def test_zero_output_layer_gives_uniform_attention(cuda_lib):
    """w3 = b3 = 0 (the reference's initialisation): every real logit is 0 and the padded ones
    must vanish from the base-2 softmax, so each sample's colour is the palette mean -- what the
    same render gives with every palette entry replaced by that mean."""
    scene, cams = make('p3d_plain', 10)
    nt, nu = synthetic.make_noise(7, 2, H, W, S)
    zero = dict(scene, w3=torch.zeros_like(scene['w3']), b3=torch.zeros_like(scene['b3']))
    mean = dict(zero, palette=scene['palette'].mean(dim=1, keepdim=True).expand_as(scene['palette']).contiguous())
    with torch.no_grad():
        a = Hh.run_cuda(zero, cams, H, W, S, nt, nu, mlp_mode=TC)
        b = Hh.run_cuda(mean, cams, H, W, S, nt, nu, mlp_mode=TC)
    assert torch.equal(a[2], b[2]) and a[2].max() > 0.5
    assert (a[0] - b[0]).abs().max().item() < 1e-6


def test_tensor_core_forward_simt_backward_matches_float64_oracle(cuda_lib):
    case, A = 'p3d_plain', 10
    scene, cams = make(case, A)
    nt, nu = synthetic.make_noise(13, 2, H, W, S)
    names = ['planes', 'w3', 'b3', 'w1', 'b1', 'w2', 'b2', 'palette', 'beta', 'alpha']
    vm_names = ['fc0_w', 'fc2_w', 'norm4_w', 'fc6_b']
    g = torch.Generator().manual_seed(1)
    wr, wm = torch.randn(2, H, W, 3, generator=g), torch.randn(2, H, W, generator=g)

    def leaves(sc, cm):
        sc = {k: (v.clone().requires_grad_() if k in names else v) for k, v in sc.items()}
        sc['view_mapper'] = {k: (v.clone().requires_grad_() if k in vm_names else v)
                             for k, v in sc['view_mapper'].items()}
        cm = dict(cm, c2w=cm['c2w'].clone().requires_grad_())
        return sc, cm, [sc[n] for n in names] + [sc['view_mapper'][n] for n in vm_names] + [cm['c2w']]

    sc, cm, lv = leaves(dbl(scene), dbl(cams))
    ref = Hh.run_oracle(sc, cm, H, W, S, nt.double(), nu.double())
    want = torch.autograd.grad((ref['rgb'] * wr.double()).sum() + (ref['mask'] * wm.double()).sum(), lv)
    dev = lambda d: {k: (v.cuda() if torch.is_tensor(v) else
                         ({a: b.cuda() for a, b in v.items()} if isinstance(v, dict) else v))
                     for k, v in d.items()}
    sc, cm, lv = leaves(dev(scene), dev(cams))
    rgb, depth, mask, _ = Hh.run_cuda(sc, cm, H, W, S, nt, nu, mlp_mode=TC)
    have = torch.autograd.grad((rgb * wr.cuda()).sum() + (mask * wm.cuda()).sum(), lv)
    assert Hh.rel_l2(rgb.detach().cpu(), ref['rgb'].float()) < 2e-4
    for n, a, b in zip(names + ['vm_' + n for n in vm_names] + ['c2w'], have, want):
        tol = 5e-3 if n in ('beta', 'alpha') else 1e-3
        assert Hh.rel_l2(a.cpu().double(), b) < tol, (n, Hh.rel_l2(a.cpu().double(), b))


def test_normals_with_a_view(cuda_lib):
    """render_normals_pipe behind the view-conditioned forward: it takes the distance row (row 0)
    of the 33-row w2."""
    scene, cams = make('p3d_plain')
    nt, nu = synthetic.make_noise(9, 2, H, W, S)
    want = Hh.run_oracle(scene, cams, H, W, S, nt, nu, compute_normals=True)
    with torch.no_grad():
        out = Hh.run_cuda(scene, cams, H, W, S, nt, nu, compute_normals=True, mlp_mode=TC)
    assert Hh.rel_l2(out[0].cpu(), want['rgb']) < 2e-4
    assert Hh.rel_l2(out[4].cpu(), want['normals']) < 1e-3
