"""The SegFormer module the fused-backbone tests bind to: the reference's ``Segformer``
(models/segformer.py) where it is installed (oracle/_ref), else a stand-in with the same module
tree, parameter names and drop-path draws, whose forward is the float64 oracle's arithmetic."""
import sys

import torch
from torch import nn

from oracle import segformer_oracle as SO


def reference_available():
    from oracle import reference_lift as RL
    from oracle import stage_encoder_reference
    return RL.available() and stage_encoder_reference.available(RL.REFERENCE_ROOT)


class _DropPath(nn.Module):
    def __init__(self, p):
        super().__init__()
        self.p = p

    def forward(self, x):
        if self.p == 0 or not self.training:
            return x
        keep = 1 - self.p
        r = x.new_empty([x.shape[0]] + [1] * (x.ndim - 1)).bernoulli_(keep)
        return x * r.div_(keep)


class _Attn(nn.Module):
    def __init__(self, C, heads, sr):
        super().__init__()
        self.num_heads, self.scale, self.sr_ratio = heads, (C // heads) ** -0.5, sr
        self.q, self.kv, self.proj = nn.Linear(C, C), nn.Linear(C, 2 * C), nn.Linear(C, C)
        if sr > 1:
            self.sr, self.norm = nn.Conv2d(C, C, sr, stride=sr), nn.LayerNorm(C)


class _DW(nn.Module):
    def __init__(self, C):
        super().__init__()
        self.dwconv = nn.Conv2d(C, C, 3, padding=1, groups=C)


class _MLP(nn.Module):
    def __init__(self, C):
        super().__init__()
        self.fc1, self.dwconv, self.gelu, self.fc2 = nn.Linear(C, 4 * C), _DW(4 * C), nn.GELU(), nn.Linear(4 * C, C)


class _Block(nn.Module):
    def __init__(self, C, heads, sr, p):
        super().__init__()
        self.norm1, self.attn = nn.LayerNorm(C, eps=1e-6), _Attn(C, heads, sr)
        self.drop_path, self.norm2, self.mlp = _DropPath(p), nn.LayerNorm(C, eps=1e-6), _MLP(C)


class _Embed(nn.Module):
    def __init__(self, cin, C, k, stride):
        super().__init__()
        self.proj, self.norm = nn.Conv2d(cin, C, k, stride=stride, padding=k // 2), nn.LayerNorm(C)


class _Linear(nn.Module):
    def __init__(self, cin, C):
        super().__init__()
        self.proj = nn.Linear(cin, C)


class StandInSegformer(nn.Module):
    def __init__(self, out_features, depths, drop_path_rate=0.1):
        super().__init__()
        self.depths = tuple(depths)
        for i in range(4):
            setattr(self, 'patch_embed%d' % (i + 1),
                    _Embed(3 if i == 0 else SO.DIMS[i - 1], SO.DIMS[i], 7 if i == 0 else 3, 4 if i == 0 else 2))
        dpr = torch.linspace(0, drop_path_rate, sum(depths)).tolist()
        cur = 0
        for i in range(4):
            setattr(self, 'block%d' % (i + 1), nn.ModuleList(
                [_Block(SO.DIMS[i], SO.HEADS[i], SO.SR[i], dpr[cur + j]) for j in range(depths[i])]))
            setattr(self, 'norm%d' % (i + 1), nn.LayerNorm(SO.DIMS[i], eps=1e-6))
            cur += depths[i]
        for i in reversed(range(4)):
            setattr(self, 'linear_c%d' % (i + 1), _Linear(SO.DIMS[i], SO.DECODER))
        self.linear_fuse = nn.Conv2d(4 * SO.DECODER, SO.DECODER, 1)
        self.linear_pred = nn.Conv2d(SO.DECODER, out_features, 1)

    def forward(self, x):
        scales = []
        for i in range(4):
            for blk in getattr(self, 'block%d' % (i + 1)):
                for _ in range(2):
                    scales.append(blk.drop_path(x.new_ones(x.shape[0], 1, 1)).reshape(-1))
        return SO.forward(dict(self.named_parameters()), self.depths, x, scales)


def make_segformer(out_features, depths, init_weights=True):
    """The reference's Segformer (or the stand-in) with these depths."""
    if reference_available():
        from oracle import reference_lift as RL
        if RL.REFERENCE_ROOT not in sys.path:
            sys.path.insert(0, RL.REFERENCE_ROOT)
        from models import segformer
        return segformer.Segformer(out_features=out_features, depths=list(depths), init_weights=init_weights)
    return StandInSegformer(out_features, depths)


def load(m, p):
    """Copies the parameter dict ``p`` (oracle names) into ``m``; returns ``m``."""
    with torch.no_grad():
        for n, t in m.named_parameters():
            t.copy_(p[n].to(t))
    return m
