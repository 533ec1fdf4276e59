"""Decoder-weight gradients of the tensor-core path (render_backward_pipe + render_wgrad_pipe) against
the fp32 SIMT kernel on the same inputs: per-tensor relative L2 and a few entries.
Usage: python tools/wgrad_check.py [B H W S R]"""
import sys, torch
sys.path.insert(0, '.')
from fixtures import synthetic
from tests import helpers as Hh
a = [int(x) for x in sys.argv[1:]] + [2, 12, 20, 16, 32][len(sys.argv) - 1:]
B, H, W, S, R = a
scene, cams = Hh.make_case('p3d_bbox', batch=B, plane_res=R, device='cuda')
nt, nu = synthetic.make_noise(13, B, H, W, S, device='cuda')
names = ['w1', 'b1', 'w2', 'b2', 'planes', 'palette']
g = torch.Generator().manual_seed(0)
wr, wm = torch.randn(B, H, W, 3, generator=g).cuda(), torch.randn(B, H, W, generator=g).cuda()
res = {}
for mode in (1, 4):
    sc = {k: (v.detach().clone().requires_grad_() if k in names else v) for k, v in scene.items()}
    rgb, depth, mask, _ = Hh.run_cuda(sc, cams, H, W, S, nt, nu, mlp_mode=mode)
    res[mode] = torch.autograd.grad((rgb * wr).sum() + (mask * wm).sum(), [sc[n] for n in names])
torch.cuda.synchronize()
for n, s_, t_ in zip(names, res[1], res[4]):
    print('%-8s rel-L2 %.3e   |simt| %.3e |tc| %.3e' % (n, Hh.rel_l2(t_, s_), s_.norm().item(), t_.norm().item()))
    if n in ('w1', 'b1', 'w2', 'b2'):
        print('   simt', s_.flatten()[:6].tolist())
        print('   tc  ', t_.flatten()[:6].tolist())
print('w2 rows tc  :', res[4][2].norm(dim=1).tolist())
print('w2 rows simt:', res[1][2].norm(dim=1).tolist())
print('w1 cols tc  :', res[4][0].norm(dim=0)[:8].tolist())
print('w1 cols simt:', res[1][0].norm(dim=0)[:8].tolist())
d = (res[4][0] - res[1][0])
print('w1 err by col :', ['%.1e' % x for x in (d.norm(dim=0) / res[1][0].norm(dim=0)).tolist()])
print('w1 err by row :', ['%.1e' % x for x in (d.norm(dim=1) / res[1][0].norm(dim=1)).tolist()[:32]])
print('w1 |col| simt :', ['%.1e' % x for x in res[1][0].norm(dim=0).tolist()])
print('w1 mean signed rel err by col:', ['%.1e' % x for x in ((d * res[1][0]).sum(0) / res[1][0].square().sum(0)).tolist()])
