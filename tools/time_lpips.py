"""Times the LPIPS-VGG loss of the inversion step at config 3's per-GPU shapes: 16 images x 16 copies
(the image and its 15 augmentations, run.py:2211-2235), prediction and target, 128^2:

  * fused: FusedLPIPS forward (saved) + backward to the prediction (nfi_lpips_forward /
    nfi_lpips_backward);
  * eager, in fp32 with TF32 off (run.py:59-60), forward + autograd.grad: the reference's module
    structure (tests/lpips_standin.py: nn.Conv2d / nn.ReLU / nn.MaxPool2d slices) and the oracle
    (oracle/lpips_oracle.py: pools by gather, ReLU by mask);
  * with the reference staged (oracle/stage_reference.py): one inversion step through render()
    (B = 16, 128^2, 64 + 64 samples per ray, synthesis fused) with the loss built as optimize_iter
    builds it (run.py:2211-2235: 15 augmented copies of cat(prediction, target), so the target side
    requires grad too), with each LPIPS.
Peak memory of each arm (torch.cuda.max_memory_allocated over one call) and the fused workspace.

CUDA events after warm-up; the two arms alternate over several rounds and the median is reported.
TFLOP/s from the shape-derived FLOP count (2 x MACs of the 13 convs: 10.02 GFLOP per image forward,
as much again for the data gradients); the bound is the 3-product bf16 rate, 989 / 3 TFLOP/s.
The card's name, power limit and SM clock are read in the same run.
Usage: python tools/time_lpips.py [steps] [rounds]   (default: 5 5)"""
import ctypes
import statistics
import subprocess
import sys
import types

import torch

sys.path.insert(0, '.')
from nerf_from_image_b200 import _lib  # noqa: E402
from nerf_from_image_b200.lpips import CONV_CHANNELS, FusedLPIPS  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import reference_lift as RL  # noqa: E402
from tests.lpips_standin import StandInLPIPSLoss, inversion_loss  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
K = int(sys.argv[1]) if len(sys.argv) > 1 else 5
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
if not torch.cuda.is_available():
    raise SystemExit('needs a GPU')
card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                       '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
print('card (name, power limit, max SM clock, SM clock):',
      card.splitlines()[0] if card else torch.cuda.get_device_name())

RES, IMAGES, COPIES = 128, 16, 16
N = IMAGES * COPIES


def conv_flops(res):
    """2 x MACs of the 13 convs on one res^2 image (the forward; the data gradients cost the same)."""
    f, level = 0, 0
    for i, (cin, cout) in enumerate(CONV_CHANNELS):
        if i in (2, 4, 7, 10):
            level += 1
        f += 2 * 9 * cin * cout * (res >> level) ** 2
    return f


def timeit(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def workspace_gb(n, save):
    q = _lib.LpipsParams()
    q.n, q.height, q.width, q.save = n, RES, RES, save
    return _lib.load().nfi_lpips_workspace_bytes(ctypes.byref(q)) / 2 ** 30


def alternate(arms, n, rounds):
    for fn in arms.values():   # warm-up: every shape the timed window uses
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timeit(fn, n))
    return {k: statistics.median(v) for k, v in times.items()}


p = LO.make_weights(seed=1)
p32 = LO.to(p, 'cuda', torch.float32)


standin = StandInLPIPSLoss(p).cuda()
fused_net = FusedLPIPS(standin)
gen = torch.Generator().manual_seed(2)
pred = (torch.rand(N, 3, RES, RES, generator=gen) * 2 - 1).cuda()
target = (torch.rand(N, 3, RES, RES, generator=gen) * 2 - 1).cuda()


def fused():
    a = pred.clone().requires_grad_()
    torch.autograd.grad(fused_net(a, target).mean(), a)


def module():
    a = pred.clone().requires_grad_()
    torch.autograd.grad(standin(a, target).mean(), a)


def oracle():
    a = pred.clone().requires_grad_()
    torch.autograd.grad(LO.distance(p32, a, target).mean(), a)


arms = {'fused': fused, 'module': module, 'oracle': oracle}
t = alternate(arms, K, ROUNDS)
mem = {k: peak_gb(fn) for k, fn in arms.items()}
fl = conv_flops(RES)
flops = N * (2 * fl + fl)   # forward of prediction and target, data gradient of the prediction
print('LPIPS-VGG, %d x %d^2 pairs (%.2f GFLOP per image forward; %.0f GFLOP per call)'
      % (N, RES, fl / 1e9, flops / 1e9))
names = {'fused': 'fused', 'module': 'eager fp32, reference module structure',
         'oracle': 'eager fp32, oracle'}
for k in arms:
    rate = flops / (t[k] * 1e-3) / 1e12
    print('  %-40s forward + backward %9.2f ms  %7.1f TFLOP/s  %5.1f %% of 989/3 TFLOP/s  peak +%.1f GB'
          % (names[k], t[k], rate, 100 * rate / (989 / 3), mem[k]))
print('  -> %.2fx over the module, %.2fx over the oracle; fused workspace %.1f GB (save = 1)'
      % (t['module'] / t['fused'], t['oracle'] / t['fused'], workspace_gb(N, 1)))

if RL.available():
    from fixtures import synthetic
    from nerf_from_image_b200 import render as R
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    torch.manual_seed(1234)
    g = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True,
                            disable_stylegan_noise=True).cuda().eval().requires_grad_(False)
    R.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                      fine_sampling=True),
                {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    R.enable_fused_inversion(g, True)
    cams = synthetic.make_cameras(1, IMAGES, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    with torch.no_grad():
        w_inv = g.mapping_network(torch.randn(IMAGES, 512, device='cuda'), None)
    tgt = target[:IMAGES]

    def step(net):
        def run():
            w = w_inv.clone().requires_grad_()
            c2w = cams['c2w'].clone().requires_grad_()
            rgb = R.render(g, RES, RES, c2w, cams['focal'], None, cams['bbox'], w, 64)[0]
            img = rgb.permute(0, 3, 1, 2) * 2 - 1
            loss = inversion_loss(net, img, tgt, COPIES - 1)
            torch.autograd.grad(loss, [w, c2w])
        return run

    steps = {'fused': step(fused_net), 'module': step(standin),
             'oracle': step(lambda a, b: LO.distance(p32, a, b)[:, None])}
    ts = alternate(steps, K, ROUNDS)
    ms = {k: peak_gb(fn) for k, fn in steps.items()}
    print('inversion step through render(), B = %d, 128^2, optimize_iter\'s loss on %d copies of each '
          'image (in1 requires grad)' % (IMAGES, COPIES))
    for k in steps:
        print('  %-40s %9.2f ms  peak +%.1f GB' % (names[k], ts[k], ms[k]))
    print('  -> %.2fx over the module, %.2fx over the oracle; fused workspace %.1f GB (save = 2)'
          % (ts['module'] / ts['fused'], ts['oracle'] / ts['fused'], workspace_gb(N, 2)))
else:
    print('inversion step through render(): not measured (reference not installed)')
print('peak memory %.1f GB' % (torch.cuda.max_memory_allocated() / 2 ** 30))
