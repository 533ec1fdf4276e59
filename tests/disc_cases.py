"""Inputs and reference modules shared by the discriminator tests (tests/test_disc_*.py) and
tools/time_discriminator.py."""
import math
import sys

import torch

from oracle import disc_oracle as DO

DATASET_CONFIG = {'camera_flipped': True}


def reference_staged():
    from oracle import reference_lift as RL
    from oracle import stage_disc_reference
    return RL.available() and stage_disc_reference.available(RL.REFERENCE_ROOT)


def reference_modules():
    """The staged reference's (discriminator, stylegan) modules, or None."""
    if not reference_staged():
        return None
    from oracle import reference_lift as RL
    if RL.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, RL.REFERENCE_ROOT)
    from models import discriminator, stylegan
    return discriminator, stylegan


def load_backbone(bb, p):
    """Copies oracle-layout parameters ``p`` into a DiscriminatorBackbone ``bb``."""
    sd = bb.state_dict()
    with torch.no_grad():
        for k, v in p.items():
            sd[k].copy_(v)
    return bb


def image(B, nc, R, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, nc, R, R, generator=g, dtype=torch.float64).to(dtype)


def cmap(B, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 512, generator=g, dtype=torch.float64).to(dtype)


def poses(B, seed, dtype=torch.float32):
    """Camera-to-world matrices [B,4,4] on a sphere of radius 2 looking at the origin, and focal
    lengths [B]."""
    g = torch.Generator().manual_seed(seed)
    az = torch.rand(B, generator=g, dtype=torch.float64) * 2 * math.pi
    el = (torch.rand(B, generator=g, dtype=torch.float64) - 0.5) * 1.0
    eye = torch.stack([torch.cos(el) * torch.cos(az), torch.cos(el) * torch.sin(az), torch.sin(el)], -1) * 2
    fwd = -eye / eye.norm(dim=-1, keepdim=True)
    up = torch.tensor([0., 0., 1.], dtype=torch.float64).expand(B, 3)
    right = torch.cross(fwd, up, dim=-1)
    right = right / right.norm(dim=-1, keepdim=True)
    up2 = torch.cross(right, fwd, dim=-1)
    m = torch.eye(4, dtype=torch.float64).repeat(B, 1, 1)
    m[:, :3, 0], m[:, :3, 1], m[:, :3, 2], m[:, :3, 3] = right, up2, -fwd, eye
    focal = 1.5 + torch.rand(B, generator=g, dtype=torch.float64)
    return m.to(dtype), focal.to(dtype)


def seed_module(m, seed):
    """Seeds every parameter of ``m`` (randn weights; biases 0.1 randn) in a fixed order."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in m.named_parameters():
            v = torch.randn(t.shape, generator=g, dtype=torch.float64)
            t.copy_(v * (0.1 if name.endswith('bias') else 1.0))
    return m


__all__ = ['DO']
