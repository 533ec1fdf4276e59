"""Times the synthesis backward to the parameters (the GAN generator step) on the GPU.

1. Full-size synthesis (512 channels, 256^2): ``FusedSynthesis.forward_trainable`` + backward
   against the module's eager fp32 forward + backward to every parameter and ws, B = 16 and 32,
   the two arms alternated, CUDA events after warm-up.
2. ``wgrad_tc_kernel`` per launch (torch.profiler, one backward at B = 32): time and achieved rate
   against the bf16 dense bound for three products per GEMM (989 / 3 TFLOP/s).
3. One G-step through ``render()`` (128^2, 64 + 64 samples, B = 32, heads on), fused generator
   step against the reference synthesis module.
Prints the card and its power limit first.  Needs the reference (oracle/_ref) for 1 and 3."""
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps=5):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def main():
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    from oracle import reference_lift as RL
    from nerf_from_image_b200.synthesis import FusedSynthesis
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RL._import_reference()
    from models import stylegan
    torch.manual_seed(0)
    net = stylegan.SynthesisNetwork(512, 256, 96).cuda().train().requires_grad_(True)
    fs = FusedSynthesis(net)
    for B in (16, 32):
        ws = torch.randn(B, net.num_ws, 512, device='cuda')
        g = torch.randn(B, 3, 256, 256, 32, device='cuda') / 256
        g_cf = g.permute(0, 1, 4, 2, 3).reshape(B, 96, 256, 256)

        def fused():
            w = ws.clone().requires_grad_()
            fs.forward_trainable(w).backward(g)

        def eager():
            w = ws.clone().requires_grad_()
            net(w).backward(g_cf)
        for f in (fused, eager):
            f()
        t = {'fused': [], 'eager': []}
        for _ in range(3):
            t['fused'].append(_time(fused, 3))
            t['eager'].append(_time(eager, 3))
        tf, te = min(t['fused']), min(t['eager'])
        print('B=%d synthesis fwd + bwd to every parameter: fused %.1f ms, eager fp32 module %.1f ms '
              '(%.1fx)' % (B, tf, te, te / tf))
    # per-layer weight-gradient GEMM
    B = 32
    ws = torch.randn(B, net.num_ws, 512, device='cuda').requires_grad_()
    g = torch.randn(B, 3, 256, 256, 32, device='cuda') / 256
    planes = fs.forward_trainable(ws)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        planes.backward(g)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if 'wgrad_tc_kernel' in e.name]
    # launches in backward order: per block from the last, ToRGB, conv1, conv0 (block 0: ToRGB, conv1)
    shapes = []
    res = [4 << i for i in range(7)]
    ch = [getattr(net, 'b%d' % r).conv1.weight.shape[0] for r in res]
    for i in range(6, -1, -1):
        shapes.append(('b%d.torgb' % res[i], 96, ch[i], 1, res[i]))
        shapes.append(('b%d.conv1' % res[i], ch[i], ch[i], 9, res[i]))
        if i:
            shapes.append(('b%d.conv0' % res[i], ch[i], ch[i - 1], 9, res[i] // 2))
    bound = 989.0 / 3
    for (name, co, ci, taps, dom), e in zip(shapes, ks):
        ms = e.device_time_total / 1e3 if hasattr(e, 'device_time_total') else e.cuda_time_total / 1e3
        flops = 2.0 * co * ci * taps * B * dom * dom
        print('%-10s Cout %3d Cin %3d taps %d K %8d: %.3f ms, %.1f TFLOP/s of products '
              '(%.0f%% of the %.0f TFLOP/s bf16 bound for 3 products)'
              % (name, co, ci, taps, B * dom * dom, ms, flops / ms / 1e9, 100 * flops / ms / 1e9 / bound, bound))
    # G-step through render()
    from fixtures import synthetic
    from nerf_from_image_b200 import render as R
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['shapenet_chairs'] if 'shapenet_chairs' in synthetic.DATASET_CONFIGS \
        else synthetic.DATASET_CONFIGS['p3d_car']
    G = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True).cuda().train()
    cams = synthetic.make_cameras(0, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    z = torch.randn(B, 512, device='cuda')
    R.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                      fine_sampling=True),
                {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    heads = ['sdf_eikonal_loss', 'total_variation_loss', 'entropy_loss']
    R.enable_fused_heads(G)

    def step():
        out = R.render(G, 128, 128, cams['c2w'], cams['focal'], None, cams['bbox'], z, 64,
                       extra_model_outputs=heads)
        mo = out[5]
        (out[0].square().mean() + sum(mo[k].mean() for k in heads)).backward()
    t = {True: [], False: []}
    for fused in (True, False):
        R.enable_fused_generator_step(G, fused)
        step()
    for _ in range(3):
        for fused in (True, False):
            R.enable_fused_generator_step(G, fused)
            t[fused].append(_time(step, 2))
    R.enable_fused_generator_step(G, False)
    print('G-step through render() (128^2, 64+64 samples, B=%d, heads): fused synthesis %.1f ms, '
          'reference synthesis %.1f ms' % (B, min(t[True]), min(t[False])))


if __name__ == '__main__':
    main()
