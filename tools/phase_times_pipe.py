"""Per-phase cycle counts of the pipelined forward kernel (timing experiment;
mlp_mode bit 0x1000 selects the DBG instantiation in which lane 0 of warp 0 of a producer set,
of the activation warpgroup and of the shading warpgroup, in CTA 0, accumulates clock64 deltas).
Modes: normal; skip_gather (producers write nothing); skip_consumer (no decoder, no field head);
window (every texel tap inside a 32 KiB window, so every load hits L1).
Usage: python tools/phase_times_pipe.py [batch] [mode ...]"""
import sys, torch
sys.path.insert(0, '.')
from nerf_from_image_b200 import fused
from fixtures import synthetic
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
MODES = {'normal': 0x1004, 'skip_gather': 0x1104, 'skip_consumer': 0x1204, 'window': 0x1804}
names = sys.argv[2:] or list(MODES)
H, W, S = 128, 128, 64
ds = synthetic.DATASET_CONFIGS['p3d_car']
sc = synthetic.make_scene(1, B, plane_res=256, scene_range=ds['scene_range'], device='cuda')
cm = synthetic.make_cameras(1, B, radius=ds['radius'], device='cuda')
nt, nu = synthetic.make_noise(1, B, H, W, S, device='cuda')
for name in names:
    cfg = fused.RenderConfig(scene_range=sc['scene_range'], mlp_mode=MODES[name])
    buf = torch.zeros(48, device='cuda')
    fused.DEBUG_BUF = buf
    with torch.no_grad():
        for _ in range(2):
            fused.fused_render(sc['planes'], sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                               sc['beta'], sc['alpha'], cm['c2w'], cm['focal'], None, None, cfg, H, W, S, nt, nu)
    torch.cuda.synchronize()
    b = buf.cpu()
    sp = max(b[9].item(), 1)
    na = max(b[16 + 9].item(), 1)
    ns = max(b[32 + 9].item(), 1)
    tiles = ns / (2 * S)
    print(name)
    print('  producer set0 warp0 (cycles per step it handled, %d steps): wait_a_free %.0f taps %.0f gather %.0f '
          'arrive %.0f' % ((sp,) + tuple((b[i] / sp).item() for i in range(4))))
    print('  activation warp0 (cycles per step, %d steps): wait_stage+slot %.0f decoder (both layers) %.0f '
          'loop %.0f | per tile: wait_cw %.0f resample %.0f' %
          ((na,) + tuple((b[16 + i] / na).item() for i in (0, 1, 2)) +
           tuple(b[16 + i].item() / tiles for i in (3, 4))))
    print('  shading warp0 (cycles per step, %d steps ~ %.1f tiles): wait_d2 %.0f ld+head %.0f store/composite %.0f '
          'loop %.0f | per tile: wait_cw %.0f resample+wait_zf %.0f tail %.0f' %
          ((ns, tiles) + tuple((b[32 + i] / ns).item() for i in (0, 1, 3, 2)) +
           tuple(b[32 + i].item() / tiles for i in (4, 5, 6))))
fused.DEBUG_BUF = None
