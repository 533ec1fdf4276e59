"""Times the GAN loop's discriminator calls, fused (nfi_disc.cu through enable_fused_discriminator)
against the eager reference module with TF32 off, at B = 32, 128^2, nc = 4, conditional pose:

  (a) the generator step's call: D frozen, forward and backward to the image;
  (b) one discriminator step without R1: D(real) and D(fake), backward to every parameter;
  (c) (b) with R1's real call (image gradient with create_graph), which runs the module in the fused
      and eager arms; a third arm, fused_r1, runs it on the kernels too
      (enable_fused_discriminator(D, r1=True): nfi_disc_backward_hvp for the penalty's backward);
  (d) a whole G/D iteration pair: the generator step through render() (fused synthesis, heads on,
      128^2, 64 + 64 samples) with D(rgb + alpha) in its loss, then a D step on real images and a
      no-grad render's fakes; with the fused D, the eager D, and no D at all (the generator step's
      loss without the discriminator term, no D step) -- the discriminator's share of the pair is
      1 - (no D) / (with D);
  (e) (d) with R1 on that D step, with the fused_r1 arm as in (c).
With --profile, one fused call of (a) and of (b), and one R1 call of the fused_r1 arm (its create_graph
backward, the HVP and the plain backward), under torch.profiler: CUDA time per kernel.

CUDA events around each step, the arms alternated, the median of the rounds; peak memory above
what was allocated before the step ((a) - (c)).  One JSON line for (a) - (c), one for (d), (e).  Needs the reference discriminator staged
(oracle/stage_disc_reference.py) and a GPU.

    python tools/time_discriminator.py [--rounds 10] [--batch 32]
"""
import argparse
import copy
import json
import re
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from nerf_from_image_b200.discriminator import enable_fused_discriminator  # noqa: E402
from tests import disc_cases as DC  # noqa: E402


def _gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                               '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--resolution', type=int, default=128)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    mods = DC.reference_modules()
    assert mods is not None, 'stage the reference discriminator first (oracle/stage_disc_reference.py)'
    dev = 'cuda:0'
    B, R, nc = args.batch, args.resolution, 4
    eager = DC.seed_module(mods[0].Discriminator(R, nc, DC.DATASET_CONFIG, conditional_pose=True), 1).to(dev)
    fused = enable_fused_discriminator(copy.deepcopy(eager))
    fused_r1 = enable_fused_discriminator(copy.deepcopy(eager), r1=True)
    pose, focal = (t.to(dev) for t in DC.poses(B, 2))
    real, fake = DC.image(B, nc, R, 3).to(dev), DC.image(B, nc, R, 4).to(dev)
    crit = lambda x, t: F.softplus(-x if t else x).mean()

    def g_call(D):
        D.requires_grad_(False)
        x = fake.clone().requires_grad_()
        crit(D(x, 0, pose, None, focal), True).backward()

    def d_step(D, r1):
        D.requires_grad_(True)
        D.zero_grad(set_to_none=True)
        x = real.clone().requires_grad_(r1)
        out = D(x, 1, pose, None, focal)
        pen = 0
        if r1:
            g, = torch.autograd.grad(out.sum(), x, create_graph=True)
            pen = g.reshape(B, -1).square().sum(dim=1).mean()
        (crit(out, True) + 2.5 * pen).backward()
        crit(D(fake, 1, pose, None, focal), False).backward()

    def r1_call(D):
        D.requires_grad_(True)
        x = real.clone().requires_grad_()
        out = D(x, 1, pose, None, focal)
        g, = torch.autograd.grad(out.sum(), x, create_graph=True)
        (crit(out, True) + 2.5 * g.reshape(B, -1).square().sum(dim=1).mean()).backward()

    rows = {'a_g_call': g_call, 'b_d_step': lambda D: d_step(D, False), 'c_d_step_r1': lambda D: d_step(D, True)}
    res = {}
    for name, fn in rows.items():
        arms = (('fused', fused), ('eager', eager)) + ((('fused_r1', fused_r1),) if name == 'c_d_step_r1' else ())
        times = {a: [] for a, _ in arms}
        peak = {}
        for arm, D in arms:   # warm-up
            fn(D)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for arm, D in arms:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(D)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1))
                peak[arm] = max(peak.get(arm, 0), torch.cuda.max_memory_allocated() - base)
        res[name] = {arm: {'median_ms': statistics.median(t), 'min_ms': min(t), 'max_ms': max(t),
                           'peak_mib': peak[arm] / 2**20} for arm, t in times.items()}
    out = {'gpu': _gpu_info(), 'batch': B, 'resolution': R, 'img_channels': nc, 'rounds': args.rounds,
           'rows': res}
    if args.profile:
        out['kernels_ms'] = {name: _profile(lambda: fn(fused)) for name, fn in list(rows.items())[:2]}
        out['kernels_ms']['r1_call'] = _profile(lambda: r1_call(fused_r1))
    print(json.dumps(out), flush=True)
    print(json.dumps({'gpu': _gpu_info(), 'batch': B, 'resolution': R, 'img_channels': nc,
                      'rows': _iteration_pairs(fused, eager, fused_r1, real, pose, focal, B,
                                               max(3, args.rounds // 2))}))


def _profile(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r'(\w+)\s*(?:<[^(]*>)?\(', e.name)
            name = m.group(1) if m else e.name[:60]
            per[name] = per.get(name, 0.0) + e.device_time_total / 1000.0
    return dict(sorted(per.items(), key=lambda kv: -kv[1])[:25])


def _iteration_pairs(fused, eager, fused_r1, real, pose, focal, B, rounds):
    """(d) and (e): G/D iteration pairs through render() with each arm's discriminator."""
    import types
    from fixtures import synthetic
    from nerf_from_image_b200 import render as Rn
    from oracle import reference_lift as RL
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    G = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True).cuda().train()
    cams = synthetic.make_cameras(0, B, ortho=cfg['ortho'], radius=cfg['radius'], with_bbox=not cfg['ortho'],
                                  device='cuda')
    z = torch.randn(B, 512, device='cuda')
    Rn.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10, fine_sampling=True),
                 {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    heads = ['sdf_eikonal_loss', 'total_variation_loss', 'entropy_loss']
    Rn.enable_fused_heads(G)
    Rn.enable_fused_generator_step(G, True)
    res_hw = real.shape[-1]

    def render(grad):
        with torch.set_grad_enabled(grad):
            out = Rn.render(G, res_hw, res_hw, cams['c2w'], cams['focal'], None, cams['bbox'], z, 64,
                            extra_model_outputs=heads if grad else [])
        rgb, alpha = out[0], out[2]
        img = torch.cat([rgb.reshape(B, res_hw, res_hw, 3), alpha.reshape(B, res_hw, res_hw, 1)], -1)
        return img.permute(0, 3, 1, 2), out[5]

    def pair(D, r1):
        G.requires_grad_(True)
        img, mo = render(True)
        loss = sum(mo[k].mean() for k in heads)
        if D is None:
            loss = loss + img.square().mean()
        else:
            D.requires_grad_(False)
            loss = loss + F.softplus(-D(img, 0, pose, None, focal)).mean()
        loss.backward()
        if D is None:
            return
        D.requires_grad_(True)
        x = real.clone().requires_grad_(r1)
        out = D(x, 1, pose, None, focal)
        pen = 0
        if r1:
            g, = torch.autograd.grad(out.sum(), x, create_graph=True)
            pen = g.reshape(B, -1).square().sum(dim=1).mean()
        (F.softplus(-out).mean() + 2.5 * pen).backward()
        fake, _ = render(False)
        F.softplus(D(fake.contiguous(), 1, pose, None, focal)).mean().backward()

    res = {}
    for name, r1 in (('d_iteration_pair', False), ('e_iteration_pair_r1', True)):
        arms = (('fused', fused), ('eager', eager)) + ((('fused_r1', fused_r1),) if r1 else ()) + (('no_d', None),)
        times = {a: [] for a, _ in arms}
        for _, D in arms:
            pair(D, r1)
        for _ in range(rounds):
            for a, D in arms:
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                pair(D, r1)
                e1.record()
                torch.cuda.synchronize()
                times[a].append(e0.elapsed_time(e1))
        row = {a: {'median_ms': statistics.median(t), 'min_ms': min(t), 'max_ms': max(t)} for a, t in times.items()}
        for a in [a for a in row if a != 'no_d']:
            row[a]['d_share'] = 1 - row['no_d']['median_ms'] / row[a]['median_ms']
        res[name] = row
    return res


if __name__ == '__main__':
    main()
