"""Float64-capable restatement of the bootstrap encoder's regression heads (the reference's
models/encoder.py:70-103 from the backbone output(s) on) in plain torch ops; in fp32 with TF32 off
it is also what the eager module computes.

    x0     = relu(interpolate(features, x4, bilinear, align_corners=False))
    a1     = relu(conv3x3(x0; post0)),  a2 = relu(conv3x3(a1; post2))
    maps   = conv3x3(a2; post4)                                    [B,4,4h,4w]
    xl     = relu(features_latent)
    al     = relu(conv3x3(xl; wpre))
    pooled = mean_{y,x} al                                         [B,C]

The heads' parameters are a dict of 'post0_w', 'post0_b', 'post2_w', 'post2_b', 'post4_w',
'post4_b', 'wpre_w', 'wpre_b' (reference layout, [Cout,Cin,3,3] and [Cout]); entries of a head the
module does not have may be missing.  Channel counts follow the tensors, so small instances serve
gradcheck.

Branch overrides (the kernel's ReLU branches): ``branches`` maps 'x0', 'a1', 'a2', 'xl', 'al' to
bool tensors of that activation's shape [B,C,H,W], standing in for ``pre-activation > 0``.
``branches_from_saved`` builds them from the fused forward's saved activations.
"""
import math

import torch
import torch.nn.functional as F

NAMES = ('post0_w', 'post0_b', 'post2_w', 'post2_b', 'post4_w', 'post4_b', 'wpre_w', 'wpre_b')


def make_params(seed=0, channels=512, maps=4, device='cpu', dtype=torch.float32):
    """Seeded random head parameters: He-normal convs (so activations keep their scale through the
    ReLUs), small biases."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for name, cout in (('post0', channels), ('post2', channels), ('post4', maps), ('wpre', channels)):
        p[name + '_w'] = torch.randn(cout, channels, 3, 3, generator=g) * math.sqrt(2.0 / (9 * channels))
        p[name + '_b'] = torch.randn(cout, generator=g) * 0.05
    return {k: v.to(device=device, dtype=dtype) for k, v in p.items()}


def params_of(enc):
    """The head parameters of a module laid out as the reference's BootstrapEncoder."""
    p = {}
    if getattr(enc, 'pose_regressor', False):
        for i in (0, 2, 4):
            p['post%d_w' % i], p['post%d_b' % i] = enc.post[i].weight, enc.post[i].bias
    if getattr(enc, 'latent_regressor', False):
        p['wpre_w'], p['wpre_b'] = enc.w_regressor_pre[0].weight, enc.w_regressor_pre[0].bias
    return p


def _relu(u, name, branches):
    m = branches[name] if branches is not None else (u > 0)
    return u * m.to(u.dtype)


def heads(p, features=None, features_latent=None, branches=None):
    """(maps [B,4,4h,4w] or None, pooled [B,C] or None) of the heads whose features are given."""
    maps = pooled = None
    if features is not None:
        up = F.interpolate(features, scale_factor=4, mode='bilinear', align_corners=False)
        x0 = _relu(up, 'x0', branches)
        a1 = _relu(F.conv2d(x0, p['post0_w'], p['post0_b'], padding=1), 'a1', branches)
        a2 = _relu(F.conv2d(a1, p['post2_w'], p['post2_b'], padding=1), 'a2', branches)
        maps = F.conv2d(a2, p['post4_w'], p['post4_b'], padding=1)
    if features_latent is not None:
        xl = _relu(features_latent, 'xl', branches)
        al = _relu(F.conv2d(xl, p['wpre_w'], p['wpre_b'], padding=1), 'al', branches)
        pooled = al.mean(dim=[2, 3])
    return maps, pooled


def pre_activations(p, features=None, features_latent=None, branches=None):
    """The pre-activations whose signs are the branches: 'x0' (the upsampled features), 'a1', 'a2'
    (post[0], post[2] outputs before their ReLU), 'xl' (features_latent), 'al' (w_regressor_pre[0]'s
    output before its ReLU), each [B,C,H,W]; with ``branches``, downstream of the given branches."""
    u = {}
    if features is not None:
        u['x0'] = F.interpolate(features, scale_factor=4, mode='bilinear', align_corners=False)
        x0 = _relu(u['x0'], 'x0', branches)
        u['a1'] = F.conv2d(x0, p['post0_w'], p['post0_b'], padding=1)
        u['a2'] = F.conv2d(_relu(u['a1'], 'a1', branches), p['post2_w'], p['post2_b'], padding=1)
    if features_latent is not None:
        u['xl'] = features_latent
        u['al'] = F.conv2d(_relu(features_latent, 'xl', branches), p['wpre_w'], p['wpre_b'], padding=1)
    return u


def branches_from_saved(saved):
    """Bool masks [B,C,H,W] from the fused forward's saved post-ReLU activations (channel-last)."""
    return {k: (v > 0).permute(0, 3, 1, 2) for k, v in saved.items()}
