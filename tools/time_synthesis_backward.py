"""Times the synthesis network's backward to the latents (the inversion setting) at the
p3d_car / cub / chairs size (512-channel StyleGAN2 synthesis, 256^2 x 96 planes):

  * fused: FusedSynthesis.forward_differentiable + backward (nfi_synthesis_forward_saved +
    nfi_synthesis_backward);
  * reference: the module in eager fp32 (TF32 off, run.py:59-60), forward + autograd.grad to ws;
  * one whole inversion step through render() (128^2 image, 64 + 64 samples per ray, gradients to
    ws and the pose) with the synthesis network fused (enable_fused_inversion) vs the module.

CUDA events after warm-up; the card's name and power limit are read in the same run.
Usage: python tools/time_synthesis_backward.py [steps] [batch ...]   (default: 5 16 32)"""
import subprocess
import sys
import types

import torch

sys.path.insert(0, '.')
from fixtures import synthetic  # noqa: E402
from oracle import reference_lift as RL  # noqa: E402
from nerf_from_image_b200 import render as R  # noqa: E402
from nerf_from_image_b200.synthesis import FusedSynthesis  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
K = int(sys.argv[1]) if len(sys.argv) > 1 else 5
BATCHES = [int(b) for b in sys.argv[2:]] or [16, 32]
if not torch.cuda.is_available():
    raise SystemExit('needs a GPU')
if not RL.available():
    raise SystemExit('reference not installed (oracle/stage_reference.py)')
card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                       '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
print('card:', card.splitlines()[0] if card else torch.cuda.get_device_name())


def timeit(fn, n):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def guarded(label, fn, n):
    try:
        ms = timeit(fn, n)
        print('%-58s %9.2f ms' % (label, ms))
        return ms
    except torch.cuda.OutOfMemoryError:
        print('%-58s out of memory' % label)
        return None
    finally:
        torch.cuda.empty_cache()


_, generator = RL._import_reference()
from models import stylegan  # noqa: E402

torch.manual_seed(1234)
net = stylegan.SynthesisNetwork(512, 256, 96).cuda().eval().requires_grad_(False)
fs = FusedSynthesis(net)

cfg = synthetic.DATASET_CONFIGS['p3d_car']
torch.manual_seed(1234)
g = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True,
                        disable_stylegan_noise=True).cuda().eval().requires_grad_(False)
R.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                  fine_sampling=True),
            {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})

for B in BATCHES:
    ws = torch.randn(B, net.num_ws, 512, device='cuda')
    gp = torch.randn(B, 3, 256, 256, 32, device='cuda')
    gp_cf = gp.permute(0, 1, 4, 2, 3).reshape(B, 96, 256, 256).contiguous()

    def fused():
        w = ws.clone().requires_grad_()
        fs.forward_differentiable(w).backward(gp)

    def reference():
        w = ws.clone().requires_grad_()
        torch.autograd.grad(net(w), w, gp_cf)

    print('B=%d' % B)
    f = guarded('  synthesis fused forward-saved + backward', fused, K)
    r = guarded('  synthesis reference eager fp32 forward + grad to ws', reference, max(2, K // 2))
    if f and r:
        print('  -> %.2fx' % (r / f))

    cams = synthetic.make_cameras(1, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    with torch.no_grad():
        w_inv = g.mapping_network(torch.randn(B, 512, device='cuda'), None)

    def step():
        w = w_inv.clone().requires_grad_()
        c2w = cams['c2w'].clone().requires_grad_()
        out = R.render(g, 128, 128, c2w, cams['focal'], None, cams['bbox'], w, 64)
        torch.autograd.grad(out[0].square().mean() + out[2].mean(), [w, c2w])

    R.enable_fused_inversion(g, True)
    f = guarded('  inversion step through render(), fused synthesis', step, K)
    R.enable_fused_inversion(g, False)
    r = guarded('  inversion step through render(), reference synthesis', step, max(2, K // 2))
    if f and r:
        print('  -> %.2fx' % (r / f))
print('peak memory %.1f GB' % (torch.cuda.max_memory_allocated() / 2 ** 30))
