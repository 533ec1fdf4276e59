"""Gradient errors at BASELINE geometry against the oracle in float64 (ground truth) and in
float32 (what the reference's autograd computes): tells a kernel error from the conditioning of
the fp32 computation itself.  Usage: python tools/grad_diag.py [case ...]"""
import sys
import torch
sys.path.insert(0, '.')
from fixtures import synthetic
from tests import helpers as Hh
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
B, H, W, S = 1, 128, 128, 64
rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()
for case in (sys.argv[1:] or ['p3d_plain', 'cub_ortho', 'p3d_bbox']):
    scene, cams = Hh.make_case(case, batch=B, plane_res=256, device='cuda')
    nt, nu = synthetic.make_noise(51, B, H, W, S, device='cuda')
    names = ['planes', 'palette', 'beta', 'alpha', 'w1', 'b1', 'w2', 'b2']
    cam_names = [k for k in ('c2w', 'focal', 'bbox', 'center') if cams[k] is not None]
    g = torch.Generator().manual_seed(0)
    wr = torch.randn(B, H, W, 3, generator=g).cuda()
    wm = torch.randn(B, H, W, generator=g).cuda()
    res = {}
    for tag in ('f64', 'f32', 'tc', 'simt'):
        cast = (lambda v: v.double()) if tag == 'f64' else (lambda v: v)
        sc = {k: (cast(v).detach().clone().requires_grad_() if k in names else
                  (cast(v) if torch.is_tensor(v) else v)) for k, v in scene.items()}
        cm = {k: (cast(v).detach().clone().requires_grad_() if k in cam_names else v)
              for k, v in cams.items()}
        if tag in ('f64', 'f32'):
            r = Hh.run_oracle(sc, cm, H, W, S, cast(nt), cast(nu))
            rgb, mask = r['rgb'], r['mask']
        else:
            if tag == 'tc':  # frozen decoder -> tensor-core backward
                for k in ('w1', 'b1', 'w2', 'b2'):
                    sc[k] = sc[k].detach()
            rgb, _, mask, _ = Hh.run_cuda(sc, cm, H, W, S, nt, nu, mlp_mode=4 if tag == 'tc' else 1)
        loss = (rgb * cast(wr)).sum() + (mask * cast(wm)).sum()
        leaves = [(n, sc[n]) for n in names if sc[n].requires_grad] + [(n, cm[n]) for n in cam_names]
        gs = torch.autograd.grad(loss, [t for _, t in leaves])
        res[tag] = dict(rgb=rgb.detach(), **{n: x.detach() for (n, _), x in zip(leaves, gs)})
    print('== %s (mask mean %.3f)' % (case, res['f32']['rgb'].abs().mean().item()))
    for n in ['rgb'] + names + cam_names:
        line = '  %-8s' % n
        for tag in ('f32', 'tc', 'simt'):
            if n in res[tag]:
                line += '  %s vs f64 %.2e' % (tag, rel(res[tag][n], res['f64'][n]))
        if n in res['tc']:
            line += '  | tc vs f32 %.2e' % rel(res['tc'][n], res['f32'][n])
        print(line)
    # where does the tensor-core kernel's plane-gradient error sit?
    gt, g64 = res['tc']['planes'].double(), res['f64']['planes']
    err = (gt - g64)
    e2 = err.square().flatten()
    top = e2.topk(1000).values.sum() / e2.sum()
    print('  planes tc: share of squared error in the 1000 worst texel-channels %.3f (of %d), max|err|/max|g| %.2e'
          % (top.item(), e2.numel(), (err.abs().max() / g64.abs().max()).item()))
    print('  per plane     :', ' '.join('%.2e' % rel(gt[:, i], g64[:, i]) for i in range(3)))
    print('  per channel/4 :', ' '.join('%.1e' % rel(gt[:, :, c:c + 4], g64[:, :, c:c + 4]) for c in range(0, 32, 4)))
    gs = res['simt']['planes'].double()
    print('  tc vs simt    : %.2e' % rel(gt, gs))
