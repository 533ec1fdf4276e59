"""Float64-capable restatement of the reference's LPIPS-VGG distance (lib/metrics.py:97-137, the
two-tensor form of ``LPIPSLoss`` over ``lpips.LPIPS(net='vgg')``) in plain torch ops; in fp32 with
TF32 off it is also the eager baseline the fused kernels are timed against.

    x'  = (x - shift) / scale                                    lpips ScalingLayer
    f_l = relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of VGG16   torchvision vgg16().features cut at
                                                                 [0:4] [4:9] [9:16] [16:23] [23:30]
    n_l = f_l / (||f_l||_channels + 1e-10)                       lpips normalize_tensor
    d   = sum_l mean_{h,w} sum_c lin_l[c] (n_l(in0) - n_l(in1))^2  NetLinLayer (1x1, no bias, eval)

The ``lpips`` package is not a dependency.  The VGG part is pinned by
tests/test_lpips_oracle.py to ``torchvision.models.vgg16(weights=None).features`` on shared random
weights (on the CPU, skipped where torchvision is absent); the scaling layer and the head are pinned
to the formulas above.  One deliberate difference: where a feature vector is entirely zero, the
gradient through its norm is 0 here (and in the kernels), where PyTorch's ``sqrt`` backward gives NaN.

Branch overrides (the kernel's branches): ``branches = (relu, pool)`` with ``relu[l]`` a bool tensor
of conv l's output shape [N,C,h,w] standing in for ``u > 0``, and ``pool[k]`` an int64 tensor
[N,C,h/2,w/2] of the window index 0..3 (row-major) standing in for the first maximum of the k-th
2x2 max pool.  ``branches_from_u`` builds them from pre-activations.
"""
import math

import torch
import torch.nn.functional as F

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CONVS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256),
         (256, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
TAPS = (1, 3, 6, 9, 12)      # conv index of relu1_2 .. relu5_3
POOLED = (1, 3, 6, 9)        # a 2x2 max pool follows these convs
EPS = 1e-10


def make_weights(seed=0, device='cpu', dtype=torch.float32):
    """Seeded random VGG16 / head weights: He-normal convs, small biases, lins |randn|."""
    g = torch.Generator().manual_seed(seed)
    p = {'shift': torch.tensor(SHIFT), 'scale': torch.tensor(SCALE), 'conv_w': [], 'conv_b': [],
         'lin': []}
    for cin, cout in CONVS:
        p['conv_w'].append(torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin)))
        p['conv_b'].append(torch.randn(cout, generator=g) * 0.05)
    for l in TAPS:
        p['lin'].append(torch.randn(CONVS[l][1], generator=g).abs())
    return to(p, device, dtype)


def to(p, device=None, dtype=None):
    f = lambda t: t.to(device=device, dtype=dtype)
    return {'shift': f(p['shift']), 'scale': f(p['scale']), 'conv_w': [f(t) for t in p['conv_w']],
            'conv_b': [f(t) for t in p['conv_b']], 'lin': [f(t) for t in p['lin']]}


def _windows(x):  # [N,C,h,w] -> [N,C,h/2,w/2,4], row-major window order
    N, C, h, w = x.shape
    return x.view(N, C, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(N, C, h // 2, w // 2, 4)


def features(p, x, branches=None, with_u=False):
    """The five taps of x [N,3,H,W] (and, with_u, every conv's pre-activation)."""
    relu_m, pool_i = branches if branches is not None else (None, None)
    sh, sc = p['shift'].view(1, 3, 1, 1), p['scale'].view(1, 3, 1, 1)
    h = (x - sh) / sc
    taps, us, k = [], [], 0
    for l in range(len(CONVS)):
        u = F.conv2d(h, p['conv_w'][l], p['conv_b'][l], padding=1)
        us.append(u)
        mask = relu_m[l] if relu_m is not None else (u > 0)
        h = u * mask.to(u.dtype)
        if l in TAPS:
            taps.append(h)
        if l in POOLED:
            win = _windows(h)
            idx = pool_i[k] if pool_i is not None else win.argmax(dim=-1)  # first maximum
            h = win.gather(-1, idx.unsqueeze(-1)).squeeze(-1)
            k += 1
    return (taps, us) if with_u else taps


def normalize(f):
    """f / (||f||_c + eps), with a zero gradient through the norm where the vector is zero."""
    s = f.square().sum(dim=1, keepdim=True)
    nz = s > 0
    r = torch.where(nz, s, torch.ones_like(s)).sqrt() * nz.to(s.dtype)
    return f / (r + EPS)


def head(p, taps0, taps1):
    d = 0
    for l in range(len(TAPS)):
        diff = (normalize(taps0[l]) - normalize(taps1[l])).square()
        d = d + (diff * p['lin'][l].view(1, -1, 1, 1)).sum(dim=1).mean(dim=[1, 2])
    return d


def distance(p, in0, in1, branches0=None, branches1=None):
    """Per-image distance [N] (the reference's [N, 1] output without its trailing axis)."""
    return head(p, features(p, in0, branches0), features(p, in1, branches1))


def branches_from_u(us):
    """(relu masks, pool indices) of pre-activations us[0..12] ([N,C,h,w] each): u > 0, and the
    first maximum of relu(u) in each window."""
    relu_m = [u > 0 for u in us]
    pool_i = [_windows(us[l].clamp_min(0)).argmax(dim=-1) for l in POOLED]
    return relu_m, pool_i
