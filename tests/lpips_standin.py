"""A stand-in for the reference's ``LPIPSLoss`` (lib/metrics.py:97-137) with the attribute layout of
``lpips.LPIPS(net='vgg')`` -- ``.lpips.scaling_layer.shift / .scale``, ``.lpips.net.slice1..5``
(torchvision's vgg16().features cut at [0:4] [4:9] [9:16] [16:23] [23:30]), ``.lpips.lins[l].model``
= (Dropout, 1x1 Conv2d without bias) -- and the reference's eager forward, built on the weights of
oracle/lpips_oracle.make_weights.  The ``lpips`` package itself is not a dependency.  Also the
inversion loop's use of it (``inversion_loss``: augmentation and the two concatenations)."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from oracle import lpips_oracle as LO


class _Scaling(nn.Module):
    def __init__(self, shift, scale):
        super().__init__()
        self.register_buffer('shift', shift.view(1, 3, 1, 1).clone())
        self.register_buffer('scale', scale.view(1, 3, 1, 1).clone())

    def forward(self, x):
        return (x - self.shift) / self.scale


class _NetLin(nn.Module):
    def __init__(self, w):
        super().__init__()
        conv = nn.Conv2d(w.numel(), 1, 1, bias=False)
        conv.weight.data.copy_(w.view(1, -1, 1, 1))
        self.model = nn.Sequential(nn.Dropout(), conv)


class _Vgg(nn.Module):
    def __init__(self, p):
        super().__init__()
        layers, i = [], 0
        for block, n in enumerate((2, 2, 3, 3, 3)):
            if block:
                layers.append(nn.MaxPool2d(2, 2))
            for _ in range(n):
                cin, cout = LO.CONVS[i]
                conv = nn.Conv2d(cin, cout, 3, padding=1)
                conv.weight.data.copy_(p['conv_w'][i])
                conv.bias.data.copy_(p['conv_b'][i])
                layers += [conv, nn.ReLU(inplace=True)]
                i += 1
        cuts = (0, 4, 9, 16, 23, 30)
        for k in range(5):
            setattr(self, 'slice%d' % (k + 1), nn.Sequential(*layers[cuts[k]:cuts[k + 1]]))

    def forward(self, x):
        out = []
        for k in range(5):
            x = getattr(self, 'slice%d' % (k + 1))(x)
            out.append(x)
        return out


class _LPIPS(nn.Module):
    def __init__(self, p):
        super().__init__()
        self.scaling_layer = _Scaling(p['shift'], p['scale'])
        self.net = _Vgg(p)
        self.lins = nn.ModuleList([_NetLin(w) for w in p['lin']])
        self.L = 5


def _normalize_tensor(x, eps=1e-10):  # lpips.normalize_tensor
    norm_factor = torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True))
    return x / (norm_factor + eps)


class StandInLPIPSLoss(nn.Module):
    """``LPIPSLoss`` with ``lpips.LPIPS(net='vgg')`` replaced by the weights of ``p``; eval, frozen."""

    def __init__(self, p):
        super().__init__()
        self.lpips = _LPIPS(LO.to(p, 'cpu', torch.float32)).eval()
        self.lpips.requires_grad_(False)

    def forward(self, in0, in1, normalize=False, reduction='none'):
        if normalize:
            in0, in1 = 2 * in0 - 1, 2 * in1 - 1
        f0 = self.lpips.net(self.lpips.scaling_layer(in0))
        f1 = self.lpips.net(self.lpips.scaling_layer(in1))
        out = sum([lin.model((_normalize_tensor(x) - _normalize_tensor(y)).square()).mean(dim=[2, 3])
                   for x, y, lin in zip(f0, f1, self.lpips.lins)])
        return out.mean() if reduction == 'mean' else out


def augment(img):
    """The inversion loop's image augmentation (run.py:720-767 with p = 1): per image a random
    rotation, scale 2^N(0, 0.2^2) and translation N(0, 0.1^2), applied with affine_grid +
    grid_sample (bilinear, zero padding).  Draws from torch's global generator on img's device."""
    bs, dev = img.shape[0], img.device
    rot = (torch.rand(bs, device=dev) - 0.5) * 2 * math.pi
    scale = torch.exp2(torch.randn(bs, device=dev) * 0.2)
    shift = torch.randn(bs, 2, device=dev) * 0.1
    c, s = torch.cos(rot), torch.sin(rot)
    mat = torch.stack([torch.stack([c * scale, -s * scale, (c * shift[:, 0] - s * -shift[:, 1]) * scale], -1),
                       torch.stack([s * scale, c * scale, (s * shift[:, 0] + c * -shift[:, 1]) * scale], -1)],
                      1)
    grid = F.affine_grid(mat.to(img.dtype), img.shape, align_corners=False)
    return F.grid_sample(img, grid, mode='bilinear', padding_mode='zeros', align_corners=False)


def inversion_loss(lpips_net, pred, target, copies=15):
    """optimize_iter's LPIPS term (run.py:2211-2235, --inv_loss vgg): the prediction and the target
    are concatenated along channels, repeated `copies` times, augmented together and split again,
    so the augmented targets carry the prediction's autograd graph (they require grad)."""
    cat = torch.cat((pred, target), dim=1).unsqueeze(1).expand(-1, copies, -1, -1, -1)
    cat = augment(cat.contiguous().flatten(0, 1))
    pred_aug = torch.cat((pred, cat[:, :3]), dim=0)
    target_aug = torch.cat((target, cat[:, 3:]), dim=0)
    return lpips_net(pred_aug, target_aug).mean() * pred.shape[0]
