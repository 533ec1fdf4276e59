"""Forward render of a view-direction-conditioned (--use_viewdir, CARLA) model at training scale:
the pipelined tensor-core kernel render_forward_pipe<VD> (NFI_MLP_AUTO) against the fp32 SIMT view
kernel (NFI_MLP_FP32_SIMT), and the pipelined kernel WITHOUT view conditioning on the same scene
as the yardstick for what layer 3 and the wider layer 2 cost.

B = 32, 128 x 128 rays, 64 + 64 samples, 256^2 planes, 10 palette entries, scene_range 3.0, white
background, view features precomputed.  The three arms are alternated in one process; the time is
that of nfi_render_forward on the stream (weight-image prep + the render kernel), CUDA events.
Usage: python tools/time_viewdir.py [batch] [rounds]"""
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from fixtures import synthetic  # noqa: E402
from nerf_from_image_b200 import fused  # noqa: E402
from tests import helpers as Hh  # noqa: E402

if not torch.cuda.is_available():
    sys.exit('time_viewdir.py needs a GPU')
B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 8
H, W, S, A = 128, 128, 64, 10


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


plain = synthetic.make_scene(21, B, plane_res=256, attention_values=A, scene_range=3.0,
                             white_background=True, object_radius=1.5, device='cuda')
view = synthetic.add_view_mapper(plain)
cm = synthetic.make_cameras(21, B, ortho=False, radius=6.4, device='cuda')
nt, nu = synthetic.make_noise(21, B, H, W, S, device='cuda')
with torch.no_grad():
    vf = Hh.view_features(view, cm, H, W).contiguous()


def render(sc, mode, with_view):
    cfg = fused.RenderConfig(scene_range=3.0, white_background=True, attention_values=A, mlp_mode=mode)
    with torch.no_grad():
        return fused.fused_render(sc['planes'], sc['w1'], sc['b1'], sc['w2'], sc['b2'], sc['palette'],
                                  sc['beta'], sc['alpha'], cm['c2w'], cm['focal'], None, None, cfg,
                                  H, W, S, nt, nu,
                                  view=(vf, sc['w3'], sc['b3']) if with_view else None)


ARMS = [('view, fp32 SIMT kernel (mlp_mode 1)', view, 1, True),
        ('view, render_forward_pipe<VD> (auto)', view, 0, True),
        ('no view, render_forward_pipe (auto)', plain, 0, False)]
outs = {}
for name, sc, mode, wv in ARMS:            # warm-up: module load, every shape
    for _ in range(2):
        outs[name] = render(sc, mode, wv)[0]
torch.cuda.synchronize()
print('card (name, power limit, SM clock now, max): %s' % card())
times = {name: [] for name, *_ in ARMS}
for _ in range(ROUNDS):                    # alternated
    for name, sc, mode, wv in ARMS:
        fused.KERNEL_EVENTS = []
        render(sc, mode, wv)
        torch.cuda.synchronize()
        (e0, e1), = fused.KERNEL_EVENTS
        times[name].append(e0.elapsed_time(e1))
fused.KERNEL_EVENTS = None
print('card after the timed rounds:                 %s' % card())
rays = B * H * W
for name, *_ in ARMS:
    t = sorted(times[name])
    med = t[len(t) // 2]
    print('%-40s median %8.2f ms (min %.2f, max %.2f) over %d  %6.2f M rays/s'
          % (name, med, t[0], t[-1], len(t), rays / med / 1e3))
a, b = outs[ARMS[1][0]], outs[ARMS[0][0]]
print('rgb, pipelined vs SIMT view kernel: rel-L2 %.2e' % ((a - b).norm() / b.norm()).item())
