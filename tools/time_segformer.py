"""Times the SegFormer-B5 backbone's forward plus backward at encoder-training size, fused
(``enable_fused_segformer``) against eager fp32 (TF32 off): CUDA events, the arms alternated,
median of the rounds; prints the card, its power limit and SM clock with the numbers.

    python tools/time_segformer.py [--batch 32] [--res 128] [--rounds 5] [--iters 5] [--profile DIR]

``--profile DIR`` instead writes a torch.profiler per-kernel table of one fused and one eager
forward plus backward to DIR.
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_from_image_b200 import segformer as FS  # noqa: E402
from oracle import segformer_oracle as SO  # noqa: E402
from tests.segformer_standin import load, make_segformer  # noqa: E402

# forward FLOP per image at 128^2 (torch.utils.flop_counter on the module, B = 1), scaled by the
# pixel count; forward plus backward is taken as 3x the forward
FWD_GFLOP_128 = 13.3


def fused_saving_gflop(res):
    """Forward GFLOP per image the fused decoder head does not do: linear_fuse (3072 -> 768) at H/4
    in the module, against its four 768 -> 768 column slices at the stages' own resolutions."""
    r0 = res // 4
    module = 2 * 3072 * 768 * r0 * r0
    fused = 2 * 768 * 768 * sum((r0 >> i) ** 2 for i in range(4))
    return (module - fused) / 1e9


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--profile', default=None)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = 'cuda:0'
    p = SO.make_params(SO.B5_DEPTHS, 512, 1, dtype=torch.float32)
    m = load(make_segformer(512, SO.B5_DEPTHS), p).to(dev).train()
    x = torch.randn(a.batch, 3, a.res, a.res, device=dev)
    g = torch.randn(a.batch, 512, a.res // 4, a.res // 4, device=dev)

    def step(fused):
        FS.enable_fused_segformer(m, enabled=fused)
        m(x).backward(g)

    for fused in (True, False):
        for _ in range(2):
            step(fused)
    torch.cuda.synchronize()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        for fused in (True, False):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(fused)
                torch.cuda.synchronize()
            table = prof.key_averages().table(sort_by='cuda_time_total', row_limit=40)
            name = 'fused' if fused else 'eager'
            with open(os.path.join(a.profile, 'segformer_%s.txt' % name), 'w') as f:
                f.write(table)
            print(name)
            print(table)
        return
    times = {True: [], False: []}
    peak = {}
    for _ in range(a.rounds):
        for fused in (True, False):
            torch.cuda.reset_peak_memory_stats()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                m.zero_grad(set_to_none=True)
                step(fused)
            e.record()
            torch.cuda.synchronize()
            times[fused].append(s.elapsed_time(e) / a.iters)
            peak[fused] = torch.cuda.max_memory_allocated() / 2 ** 30
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    module_gflop = FWD_GFLOP_128 * (a.res / 128) ** 2
    tflop = {False: 3 * module_gflop * a.batch / 1e3,                                   # the module's ops
             True: 3 * (module_gflop - fused_saving_gflop(a.res)) * a.batch / 1e3}     # the fused arm's own
    print(card())
    for fused, name in ((True, 'fused'), (False, 'eager fp32')):
        rate = tflop[fused] / (med[fused] / 1e3)
        print('%-10s B %d %d^2: forward+backward %.1f ms (rounds %s), %.2f TFLOP of its own ops, %.1f TFLOP/s '
              '(%.1f %% of 989/3), peak %.2f GiB' % (name, a.batch, a.res, med[fused],
                                                     ' '.join('%.1f' % t for t in times[fused]), tflop[fused], rate,
                                                     100 * rate / (989 / 3), peak[fused]))
    print('eager / fused: %.2fx' % (med[False] / med[True]))


if __name__ == '__main__':
    main()
