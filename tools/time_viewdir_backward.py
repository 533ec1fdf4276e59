"""Inversion backward of a view-direction-conditioned (--use_viewdir, CARLA) model at training
scale: the pipelined tensor-core kernel render_backward_pipe<VD> (NFI_MLP_AUTO) against the fp32
SIMT view kernel (NFI_MLP_FP32_SIMT), and the plain render_backward_pipe WITHOUT view conditioning
on the same scene as the yardstick for what the view costs.

Scene of tools/time_viewdir.py: B = 32, 128 x 128 rays, 64 + 64 samples, 256^2 planes, 10 palette
entries, scene_range 3.0, white background, view features precomputed.  Gradients to the planes,
palette, beta / alpha, the pose (c2w, focal) and the view features; decoder and mapper frozen.  The
three arms are alternated in one process; the time is that of nfi_render_backward on the stream
(weight-image prep + the backward kernel), CUDA events around the call.
Usage: python tools/time_viewdir_backward.py [batch] [rounds]"""
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from fixtures import synthetic  # noqa: E402
from nerf_from_image_b200 import _lib, fused  # noqa: E402
from tests import helpers as Hh  # noqa: E402

if not torch.cuda.is_available():
    sys.exit('time_viewdir_backward.py needs a GPU')
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


# CUDA events around every nfi_render_backward call of the binding
lib = _lib.load()
EVENTS = []
_bwd = lib.nfi_render_backward


def timed_backward(*args):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = _bwd(*args)
    e1.record()
    EVENTS.append((e0, e1))
    return rc


lib.nfi_render_backward = timed_backward

plain = synthetic.make_scene(21, B, plane_res=256, attention_values=A, scene_range=3.0,
                             white_background=True, object_radius=1.5, device='cuda')
view = synthetic.add_view_mapper(plain)
cm = synthetic.make_cameras(21, B, ortho=False, radius=6.4, device='cuda')
nt, nu = synthetic.make_noise(21, B, H, W, S, device='cuda')
with torch.no_grad():
    vf = Hh.view_features(view, cm, H, W).contiguous()
g = torch.Generator(device='cuda').manual_seed(0)
wr = torch.randn(B, H, W, 3, device='cuda', generator=g)


def backward(sc, mode, with_view):
    cfg = fused.RenderConfig(scene_range=3.0, white_background=True, attention_values=A, mlp_mode=mode)
    leaves = [sc['planes'].clone().requires_grad_(), sc['palette'].clone().requires_grad_(),
              sc['beta'].clone().requires_grad_(), sc['alpha'].clone().requires_grad_(),
              cm['c2w'].clone().requires_grad_(), cm['focal'].clone().requires_grad_()]
    vfl = vf.clone().requires_grad_()
    planes, palette, beta, alpha, c2w, focal = leaves
    rgb = fused.fused_render(planes, sc['w1'], sc['b1'], sc['w2'], sc['b2'], palette, beta, alpha,
                             c2w, focal, None, None, cfg, H, W, S, nt, nu,
                             view=(vfl, sc['w3'], sc['b3']) if with_view else None)[0]
    return torch.autograd.grad((rgb * wr).sum(), leaves + ([vfl] if with_view else []))


ARMS = [('view, fp32 SIMT kernel (mlp_mode 1)', view, 1, True),
        ('view, render_backward_pipe<VD> (auto)', view, 0, True),
        ('no view, render_backward_pipe (auto)', plain, 0, False)]
outs = {}
for name, sc, mode, wv in ARMS:            # warm-up: module load, every shape
    for _ in range(2):
        outs[name] = backward(sc, mode, wv)
torch.cuda.synchronize()
print('card (name, power limit, SM clock now, max): %s' % card())
times = {name: [] for name, *_ in ARMS}
for _ in range(ROUNDS):                    # alternated
    for name, sc, mode, wv in ARMS:
        EVENTS.clear()
        backward(sc, mode, wv)
        torch.cuda.synchronize()
        (e0, e1), = EVENTS
        times[name].append(e0.elapsed_time(e1))
print('card after the timed rounds:                 %s' % card())
for name, *_ in ARMS:
    t = sorted(times[name])
    print('%-40s median %8.2f ms (min %.2f, max %.2f) over %d' % (name, t[len(t) // 2], t[0], t[-1], len(t)))
a, b = outs[ARMS[1][0]], outs[ARMS[0][0]]
for n, x, y in zip(('planes', 'palette', 'beta', 'alpha', 'c2w', 'focal', 'view_features'), a, b):
    print('%-14s pipelined vs SIMT view kernel: rel-L2 %.2e' % (n, ((x - y).norm() / y.norm()).item()))
