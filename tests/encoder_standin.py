"""A module laid out as the reference's ``BootstrapEncoder`` (models/encoder.py:21-103) for tests
that run where the reference is not installed: the same attribute names, head layout and forward,
with a one-conv stand-in for the SegFormer backbone (a stride-4 conv, so features are 1/4 of the
image like SegFormer's).  Where the reference is installed (oracle/_ref), ``reference_encoder``
builds the real module instead."""
import sys

import torch
import torch.nn.functional as F
from torch import nn


class FixedFeatures(nn.Module):
    """A backbone that returns given features whatever the image."""

    def __init__(self, features):
        super().__init__()
        self.features = features

    def forward(self, x):
        return self.features


class StandInBootstrapEncoder(nn.Module):

    def __init__(self, latent_dim, pose_regressor=True, latent_regressor=True, separate_backbones=False):
        super().__init__()
        self.backbone = nn.Conv2d(3, 512, 4, stride=4)
        if separate_backbones:
            self.backbone_latent = nn.Conv2d(3, 512, 4, stride=4)
        self.pose_regressor = pose_regressor
        self.latent_regressor = latent_regressor
        self.separate_backbones = separate_backbones
        if pose_regressor:
            self.post = nn.Sequential(
                nn.Conv2d(512, 512, 3, padding=1), nn.ReLU(inplace=True),
                nn.Conv2d(512, 512, 3, padding=1), nn.ReLU(inplace=True),
                nn.Conv2d(512, 4, 3, padding=1))
        if latent_regressor:
            self.w_regressor_pre = nn.Sequential(nn.Conv2d(512, 512, 3, padding=1), nn.ReLU(inplace=True))
            self.w_regressor_post = nn.Sequential(
                nn.Linear(512, 512), nn.ReLU(inplace=True), nn.Linear(512, latent_dim), nn.LeakyReLU(0.2))

    def forward(self, x):
        features = self.backbone(x)
        coords = segmentation = w = None
        if self.pose_regressor:
            up = F.relu(F.interpolate(features, scale_factor=4, mode='bilinear', align_corners=False))
            maps = self.post(up)
            coords = maps[:, :3].permute(0, 2, 3, 1)
            segmentation = torch.sigmoid(maps[:, 3])
        if self.latent_regressor:
            fl = self.backbone_latent(x) if self.separate_backbones else features
            w = self.w_regressor_post(self.w_regressor_pre(F.relu(fl)).mean(dim=[2, 3])).unsqueeze(1)
        return coords, segmentation, w


def reference_encoder(latent_dim, pose_regressor=True, latent_regressor=True, separate_backbones=False):
    """The staged reference's BootstrapEncoder (random init, pretrained=False), or None."""
    from oracle import reference_lift as RL
    from oracle import stage_encoder_reference
    if not (RL.available() and stage_encoder_reference.available(RL.REFERENCE_ROOT)):
        return None
    if RL.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, RL.REFERENCE_ROOT)
    from models import encoder
    return encoder.BootstrapEncoder(latent_dim, pose_regressor=pose_regressor,
                                    latent_regressor=latent_regressor,
                                    separate_backbones=separate_backbones, pretrained=False)


def load_params(enc, p, post_seed=0):
    """Copies oracle-layout head parameters ``p`` into ``enc`` and seeds w_regressor_post."""
    from oracle import encoder_oracle as EO
    with torch.no_grad():
        for k, v in EO.params_of(enc).items():
            v.copy_(p[k])
    if getattr(enc, 'latent_regressor', False):
        seed_linear(enc.w_regressor_post, post_seed)
    return enc


def seed_linear(seq, seed):
    """Seeded random weights for the Linear layers of ``seq`` (w_regressor_post)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in seq:
            if isinstance(m, nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) / m.in_features ** 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.05)
    return seq
