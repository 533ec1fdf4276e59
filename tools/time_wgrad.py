"""Times the tensor-core backward kernels of the GAN generator step at config-2 geometry: backward()
with only the decoder weights requiring grad (render_wgrad_pipe alone), only planes + palette
(render_backward_pipe alone), both in ONE sweep (render_wgrad_pipe<PLANES>, the default) and both
as two sweeps (debug bit 0x2000 of mlp_mode).  Usage: python tools/time_wgrad.py [batch]"""
import sys, torch
sys.path.insert(0, '.')
from nerf_from_image_b200 import fused
from fixtures import synthetic
B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
H, W, S = 128, 128, 64
ds = synthetic.DATASET_CONFIGS['p3d_car']
sc = synthetic.make_scene(1, B, plane_res=256, scene_range=ds['scene_range'], device='cuda')
cm = synthetic.make_cameras(1, B, radius=ds['radius'], device='cuda')
nt, nu = synthetic.make_noise(1, B, H, W, S, device='cuda')
cfg1 = fused.RenderConfig(scene_range=sc['scene_range'])
cfg2 = fused.RenderConfig(scene_range=sc['scene_range'], mlp_mode=0x2000)
ev = lambda: torch.cuda.Event(enable_timing=True)
for label, wg, pl, cfg in (('weights only (render_wgrad_pipe)', True, False, cfg1),
                           ('planes + palette only (render_backward_pipe)', False, True, cfg1),
                           ('both, one sweep (render_wgrad_pipe<PLANES>)', True, True, cfg1),
                           ('both, two sweeps', True, True, cfg2)):
    t = {k: v.clone().requires_grad_(wg) for k, v in sc.items() if k in ('w1', 'b1', 'w2', 'b2')}
    planes = sc['planes'].clone().requires_grad_(pl)
    pal = sc['palette'].clone().requires_grad_(pl)
    ms = []
    for it in range(5):
        rgb, depth, mask, _ = fused.fused_render(planes, t['w1'], t['b1'], t['w2'], t['b2'], pal, sc['beta'],
                                                 sc['alpha'], cm['c2w'], cm['focal'], None, None, cfg, H, W, S, nt, nu)
        loss = rgb.square().mean() + mask.mean()
        a, b = ev(), ev()
        a.record(); loss.backward(); b.record()
        torch.cuda.synchronize()
        if it >= 2: ms.append(a.elapsed_time(b))
        for x in list(t.values()) + [planes, pal]: x.grad = None
    print('%-48s backward() %.2f ms at B=%d' % (label, sum(ms) / len(ms), B))
