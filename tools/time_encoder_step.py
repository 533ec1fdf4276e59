"""Times encoder training (train_coord_regressor, run.py:1521-1706) on the GPU, B = 32, 128^2:

(a) the regression heads forward + backward (gradients to the features and every head weight):
    the fused heads against the eager fp32 heads (the module's ops, TF32 off), with the achieved
    rate from the shape arithmetic and its share of the bf16 dense bound for three products per
    GEMM (989 / 3 TFLOP/s);
(b) one encoder step (SegFormer backbone, heads, criteria, backward, Adam) of the reference
    BootstrapEncoder in three arms: the heads fused ('heads'), the backbone and the heads fused
    ('full'), and eager; and the backbone's own forward + backward, eager and fused;
(c) one whole iteration: (b) after the no-grad generator render with compute_coords=True (fused
    synthesis and render), in the same three arms;
(d) the peak memory of each arm.
Arms alternate within each round (CUDA events, every shape warmed up first); the median of the
rounds is printed.  The card's name, power limit and SM clock are read in the same call.  Needs the
reference (oracle/_ref) for (b) and (c)."""
import os
import statistics
import subprocess
import sys
import types

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, R, LAT, ROUNDS = 32, 128, 512, 5
BOUND = 989.0 / 3   # TFLOP/s: bf16 dense, three products per GEMM


def head_flops(B, h, w, C=512):
    """Forward + data and weight gradients of the four head convs (2 x 9 Cin Cout per position)."""
    H, W = 4 * h, 4 * w
    fwd = 2 * 9 * C * (C + C + 4) * H * W + 2 * 9 * C * C * h * w
    return 3.0 * fwd * B


def _time(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def _peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def alternate(arms, reps=3, rounds=ROUNDS):
    """{name: (median ms, peak GB)} of the arms, alternated in every round after one warm-up each."""
    peaks = {k: _peak_gb(f) for k, f in arms.items()}
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            t[k].append(_time(f, reps))
    return {k: (statistics.median(v), peaks[k]) for k, v in t.items()}


def main():
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from nerf_from_image_b200.encoder import enable_fused_encoder, heads
    from nerf_from_image_b200.segformer import enable_fused_segformer
    from oracle import encoder_oracle as EO
    from tests.encoder_standin import StandInBootstrapEncoder, load_params, reference_encoder

    # (a) the heads
    h = w = R // 4
    enc = load_params(StandInBootstrapEncoder(LAT), EO.make_params(seed=1)).cuda().train()
    g = torch.Generator().manual_seed(2)
    f = torch.randn(B, 512, h, w, generator=g).cuda()
    gm = torch.randn(B, R, R, 4, generator=g).cuda()
    gp = torch.randn(B, 512, generator=g).cuda()
    p = EO.params_of(enc)

    def fused_heads():
        a = f.clone().requires_grad_()
        maps, pooled = heads(enc, a, a)
        ((maps * gm).sum() + (pooled * gp).sum()).backward()

    def eager_heads():
        a = f.clone().requires_grad_()
        maps, pooled = EO.heads(p, a, a)
        ((maps.permute(0, 2, 3, 1) * gm).sum() + (pooled * gp).sum()).backward()

    res = alternate({'fused': fused_heads, 'eager': eager_heads})
    fl = head_flops(B, h, w)
    for k, (ms, gb) in res.items():
        print('(a) heads fwd + bwd, B=%d %d^2, %-5s: %.2f ms, %.1f TFLOP/s (%.0f%% of %.0f), peak %.2f GB'
              % (B, R, k, ms, fl / ms / 1e9, 100 * fl / ms / 1e9 / BOUND, BOUND, gb))
    print('    (%.2f TFLOP of products per call from the shapes)' % (fl / 1e12))
    del enc, f, gm, gp, p
    torch.cuda.empty_cache()

    # (b) one encoder step on the reference BootstrapEncoder
    torch.manual_seed(3)
    base = reference_encoder(LAT)
    if base is None:
        raise SystemExit('(b), (c) need the reference (oracle/_ref): run __graft_entry__.build()')
    state = base.state_dict()
    img = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).cuda()
    tc, tm = torch.randn(B, R, R, 3, generator=g).cuda(), (torch.rand(B, R, R, generator=g) > 0.5).float().cuda()
    tw = torch.randn(B, 1, LAT, generator=g).cuda()
    models = {}
    for name in ('heads', 'full', 'eager'):
        m = reference_encoder(LAT)
        m.load_state_dict(state)
        if name != 'eager':
            enable_fused_encoder(m)
        if name == 'full':
            enable_fused_segformer(m.backbone)
        model = nn.DataParallel(m.cuda(), [0])
        model.requires_grad_(True)
        model.train()
        models[name] = (model, torch.optim.Adam(model.parameters(), lr=6e-5))

    def step(name, x=None):
        model, opt = models[name]
        opt.zero_grad()
        c, s, wp = model(img if x is None else x)
        loss = ((c - tc).norm(dim=-1).mul(tm).mean() + nn.L1Loss()(s, tm) + nn.MSELoss()(wp, tw))
        loss.backward()
        opt.step()

    gfeat = torch.randn(B, 512, h, w, generator=g).cuda()
    bb = {k: models[k][0].module.backbone for k in ('eager', 'full')}

    res = alternate({'heads': lambda: step('heads'), 'full': lambda: step('full'), 'eager': lambda: step('eager'),
                     'backbone eager': lambda: bb['eager'](img).backward(gfeat),
                     'backbone fused': lambda: bb['full'](img).backward(gfeat)})
    for k in ('backbone eager', 'backbone fused'):
        print('(b) SegFormer-B5 forward + backward, B=%d %d^2, %-5s: %.1f ms, peak %.2f GB'
              % (B, R, k.split()[1], *res[k]))
    for k, what in (('heads', 'heads fused'), ('full', 'backbone + heads fused'), ('eager', 'eager')):
        ms, gb = res[k]
        print('(b) encoder step, B=%d %d^2, %-22s: %.1f ms, peak %.2f GB' % (B, R, what, ms, gb))

    # (c) the whole iteration: the no-grad generator render with coords, then the encoder step
    from fixtures import synthetic
    from nerf_from_image_b200 import render as RR
    from oracle import reference_lift as RL
    _, generator = RL._import_reference()
    cfg = synthetic.DATASET_CONFIGS['p3d_car']
    G = generator.Generator(512, cfg['scene_range'], attention_values=10, use_sdf=True).cuda().eval()
    cams = synthetic.make_cameras(0, B, ortho=cfg['ortho'], radius=cfg['radius'], with_bbox=not cfg['ortho'],
                                  device='cuda')
    RR.configure(types.SimpleNamespace(use_viewdir=False, use_sdf=True, attention_values=10, fine_sampling=True),
                 {'scene_range': cfg['scene_range'], 'white_background': cfg['white_background']})
    RR.enable_fused_synthesis(G)
    RR.enable_fused_heads(G)
    z = torch.randn(B, 512, device='cuda')

    def iteration(name):
        with torch.no_grad():
            out = RR.render(G, R, R, cams['c2w'], cams['focal'], None, cams['bbox'], z, 64,
                            compute_coords=True)
            x = out[0].clamp(-1, 1).permute(0, 3, 1, 2)
        step(name, x)

    res = alternate({k: (lambda k=k: iteration(k)) for k in ('heads', 'full', 'eager')}, reps=2)
    for k, what in (('heads', 'heads fused'), ('full', 'backbone + heads fused'), ('eager', 'eager')):
        ms, gb = res[k]
        print('(c) train_coord_regressor iteration (render with coords + encoder step), B=%d %d^2, %-22s: '
              '%.1f ms, peak %.2f GB' % (B, R, what, ms, gb))


if __name__ == '__main__':
    main()
