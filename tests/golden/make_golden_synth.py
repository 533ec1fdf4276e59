"""Golden vectors of the tri-plane producer, made by the UNMODIFIED reference
``models.stylegan.SynthesisNetwork`` (models/stylegan.py:438-490 of the reference checkout that
oracle/reference_lift.py finds):  python tests/golden/make_golden_synth.py

Small networks (8^2 planes, <= 64 channels, w_dim 128) so that the parameters themselves
fit in the fixture (each file stays under 1 MB): the kernels are checked against these files
(tests/test_synthesis_gpu.py) wherever the reference is not installed.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import reference_lift as RL  # noqa: E402
from oracle import synthesis_oracle as SO  # noqa: E402

CASES = {
    # name: (seed, img_resolution, channel_base, channel_max, batch, noise_mode)
    'synth_c64_const': (11, 8, 2048, 64, 2, 'const'),
    'synth_mixed_nonoise': (12, 8, 256, 64, 3, None),
}


def build(seed, res, cbase, cmax, noise):
    RL._import_reference()
    from models import stylegan
    torch.manual_seed(seed)
    net = stylegan.SynthesisNetwork(128, res, 96, channel_base=cbase, channel_max=cmax).eval()
    with torch.no_grad():
        for n, p in net.named_parameters():
            if n.endswith('bias') and 'affine' not in n:
                p.normal_(0, 0.2)
            if n.endswith('noise_strength'):
                p.fill_(0.1 if noise else 0.0)
    if noise is None:
        for m in net.modules():
            if hasattr(m, 'use_noise'):
                m.use_noise = False
    return net


def main():
    out_dir = os.path.join(HERE, 'synth')
    os.makedirs(out_dir, exist_ok=True)
    for name, (seed, res, cbase, cmax, B, noise) in CASES.items():
        net = build(seed, res, cbase, cmax, noise)
        ws = torch.randn(B, net.num_ws, 128)
        with torch.no_grad():
            img = net(ws, noise_mode=noise or 'const')
        p = SO.extract_params(net)
        meta = p.pop('meta')
        arrays = {'param:' + k: v.numpy() for k, v in p.items() if not k.endswith('resample_filter')}
        arrays['ws'] = ws.numpy()
        arrays['img'] = img.numpy()
        arrays['meta_resolutions'] = np.array(meta['resolutions'])
        arrays['meta_use_noise'] = np.array([int(v['use_noise']) for v in meta['layers'].values()])
        arrays['meta_layers'] = np.array(list(meta['layers'].keys()))
        arrays['meta_dims'] = np.array([meta['img_resolution'], meta['img_channels'], meta['w_dim']])
        arrays['noise_mode'] = np.array(noise or 'none')
        np.savez_compressed(os.path.join(out_dir, name + '.npz'), **arrays)
        print(name, 'img', tuple(img.shape), 'mean |img| %.3f' % img.abs().mean().item())


if __name__ == '__main__':
    main()
