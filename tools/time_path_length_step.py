"""Times the path-length regulariser's double backward (the generator step of the documented
recipe, --path_length_regularization) on the GPU.

1. Full-size synthesis (512 channels, 256^2), B = 16 and 32: forward + VJP (pl_grad) + HVP +
   parameter backward through ``FusedSynthesis.forward_trainable_with_path_length`` against the
   module's eager fp32 forward + create_graph grad + backward, the two arms alternated, CUDA
   events after warm-up.
2. The HVP's kernels (torch.profiler, one fused step at B = 32): total time per kernel name.
3. One path-length G-step through ``render()`` (128^2, 64 + 64 samples, B = 32, heads on) with
   ``enable_fused_path_length`` against today's route (the reference synthesis module).
Prints the card and its power limit first.  Needs the reference (oracle/_ref)."""
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps=3):
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

        def fused():
            w = ws.clone().requires_grad_()
            planes, pl_grad = fs.forward_trainable_with_path_length(w)
            ((planes * g).sum() + pl_grad.square().sum()).backward()

        def eager():
            w = ws.clone().requires_grad_()
            img = net(w)
            planes = img.view(B, 3, 32, 256, 256)
            pl_noise = torch.randn_like(planes) / 256
            gw, = torch.autograd.grad((planes * pl_noise).sum(), w, create_graph=True)
            ((img.view(B, 3, 32, 256, 256).permute(0, 1, 3, 4, 2) * g).sum() + gw.square().sum()).backward()
        for f in (fused, eager):
            f()
        t = {'fused': [], 'eager': []}
        for _ in range(3):
            t['fused'].append(_time(fused))
            t['eager'].append(_time(eager))
        net.zero_grad(set_to_none=True)
        print('B=%d synthesis forward + VJP + HVP + parameter backward: fused %s ms, eager fp32 %s ms'
              % (B, ' '.join('%.1f' % x for x in t['fused']), ' '.join('%.1f' % x for x in t['eager'])))

    # 2. the kernels of one fused step at B = 32
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fused()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name == 'CUDA':
            k = e.name.split('(')[0][:60]
            n, s = tot.get(k, (0, 0.0))
            tot[k] = (n + 1, s + e.device_time_total / 1000)
    print('B=32 fused step, kernels by total time (ms):')
    for k, (n, s) in sorted(tot.items(), key=lambda kv: -kv[1][1])[:16]:
        print('  %-60s %4d launches %8.2f ms' % (k, n, s))
    del net, fs
    torch.cuda.empty_cache()

    # 3. one path-length G-step through render()
    from fixtures import synthetic
    from nerf_from_image_b200 import render as R
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    torch.manual_seed(1)
    gen = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True).cuda()
    gen.train().requires_grad_(True)
    B, H = 32, 128
    cams = synthetic.make_cameras(1, B, ortho=cfg['ortho'], radius=cfg['radius'],
                                  with_bbox=not cfg['ortho'], device='cuda')
    z = torch.randn(B, 512, device='cuda')
    R.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10,
                                      fine_sampling=True),
                {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    req = ['sdf_eikonal_loss', 'total_variation_loss', 'entropy_loss', 'path_length']

    def step():
        out = R.render(gen, H, H, cams['c2w'], cams['focal'], None, cams['bbox'], z, 64,
                       extra_model_outputs=req)
        mo = out[5]
        loss = out[0].square().mean() + 0.1 * mo['sdf_eikonal_loss'].mean() \
            + mo['total_variation_loss'].mean() + 0.01 * mo['entropy_loss'].mean() \
            + (mo['path_length'] - 1.0).square().mean()
        loss.backward()
        gen.zero_grad(set_to_none=True)
    R.enable_fused_generator_step(gen)
    R.enable_fused_heads(gen)
    t = {True: [], False: []}
    for fused_pl in (True, False):
        R.enable_fused_path_length(gen, fused_pl)
        step()
    for _ in range(3):
        for fused_pl in (True, False):
            R.enable_fused_path_length(gen, fused_pl)
            t[fused_pl].append(_time(step, 2))
    print('path-length G-step through render() (128^2, 64+64 samples, B=32, heads): '
          'fused path length %s ms, reference synthesis module %s ms'
          % (' '.join('%.1f' % x for x in t[True]), ' '.join('%.1f' % x for x in t[False])))


if __name__ == '__main__':
    main()
