"""Regulariser heads of the generator on the sm_90a point evaluator.

/root/reference/models/generator.py:520-585: on (nstrata-1)^3 stratified points per image the
first decoder output d(x) and its spatial gradient feed the eikonal, distance, total-variation
and entropy terms of the GAN generator step / the SDF pre-training loop (run.py:824-868,1007-1044).
The reference gets grad_x d with ``torch.autograd.grad(create_graph=True)`` through the unfused
decoder and a hand-written twice-differentiable grid sample (lib/ops.py:58-120); here

    SdfPoints.apply(planes, w1, b1, w2, b2, points, scene_range, layout) -> (d [B,N], g [B,N,3])

is ONE kernel (nfi_sdf_points_forward) and its backward -- gradients of both outputs to the
planes and the decoder, second-order terms analytic -- one more (nfi_sdf_points_backward).
``regulariser_heads`` then forms the four losses exactly as the reference does, with the same
two random draws in the same order (``torch.rand_like`` of lib/ops.py:23, ``torch.randn_like`` of
generator.py:554), so a seeded run consumes the RNG identically.
"""
import ctypes

import torch

from . import _lib
from .fused import planes_from_channel_last, planes_to_channel_last


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class SdfPoints(torch.autograd.Function):
    """(planes, w1 [64,32], b1 [64], w2 [1+A,64], b2 [1+A], points [B,N,3] world units) ->
    (d [B,N] first decoder output, g [B,N,3] = d d / d point).  Differentiable in planes and the
    decoder parameters (through both outputs), not in the points (the reference's stratified
    points are constants: generator.py:523-536 takes the gradient w.r.t. them only to FORM g)."""

    @staticmethod
    def forward(ctx, planes, w1, b1, w2, b2, points, scene_range, layout, want_grad):
        lib = _lib.load()
        if not planes.is_cuda:
            raise _lib.NfiError('the fused heads only run on CUDA tensors (there is no CPU path)')
        dev = planes.device
        f32 = lambda t: t.detach().to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            planes_cl = f32(planes) if layout == 'channel_last' else planes_to_channel_last(planes.detach())
            w1c, b1c, w2c, b2c, pts = f32(w1), f32(b1), f32(w2), f32(b2), f32(points)
            B, N = pts.shape[0], pts.shape[1]
            assert pts.shape == (B, N, 3) and planes_cl.shape[0] == B, (pts.shape, planes_cl.shape)
            d = torch.empty(B, N, device=dev)
            g = torch.empty(B, N, 3, device=dev) if want_grad else None
            p = SdfPoints._params(planes_cl, w1c, b1c, w2c, b2c, pts, scene_range)
            p.d, p.grad = _ptr(d), _ptr(g)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.nfi_sdf_points_forward(ctypes.byref(p), stream))
        ctx.scene_range, ctx.layout = float(scene_range), layout
        ctx.save_for_backward(planes_cl, w1c, b1c, w2c, b2c, pts)
        if g is None:
            g = torch.empty(0, device=dev)
            ctx.mark_non_differentiable(g)
        return d, g

    @staticmethod
    def _params(planes_cl, w1, b1, w2, b2, pts, scene_range):
        p = _lib.SdfPointsParams()
        p.batch, p.plane_res = planes_cl.shape[0], planes_cl.shape[2]
        p.scene_range, p.n_points = float(scene_range), pts.shape[1]
        p.planes, p.w1, p.b1, p.w2, p.b2, p.points = (_ptr(planes_cl), _ptr(w1), _ptr(b1), _ptr(w2),
                                                       _ptr(b2), _ptr(pts))
        return p

    @staticmethod
    def backward(ctx, g_d, g_g):
        planes_cl, w1, b1, w2, b2, pts = ctx.saved_tensors
        lib = _lib.load()
        dev = planes_cl.device
        n_planes, n_w1, n_b1, n_w2, n_b2 = ctx.needs_input_grad[:5]
        with torch.cuda.device(dev):
            p = SdfPoints._params(planes_cl, w1, b1, w2, b2, pts, ctx.scene_range)
            g = _lib.SdfPointsGrads()
            g_d = g_d.to(torch.float32).contiguous() if g_d is not None else None
            g_g = g_g.to(torch.float32).contiguous() if (g_g is not None and g_g.numel() > 0) else None
            if g_d is None and g_g is None:
                return (None,) * 9
            g.g_d, g.g_grad = _ptr(g_d), _ptr(g_g)
            gp = torch.zeros_like(planes_cl) if n_planes else None
            wgrad = n_w1 or n_b1 or n_w2 or n_b2
            gw1 = torch.zeros_like(w1) if wgrad else None
            gb1 = torch.zeros_like(b1) if wgrad else None
            gw2 = torch.zeros_like(w2) if wgrad else None     # only row 0 receives a gradient
            gb2 = torch.zeros_like(b2) if wgrad else None
            g.grad_planes, g.grad_w1, g.grad_b1 = _ptr(gp), _ptr(gw1), _ptr(gb1)
            g.grad_w2_row0, g.grad_b2_0 = _ptr(gw2), _ptr(gb2)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.nfi_sdf_points_backward(ctypes.byref(p), ctypes.byref(g), stream))
            if n_planes and ctx.layout != 'channel_last':
                gp = planes_from_channel_last(gp)
        return (gp if n_planes else None, gw1 if n_w1 else None, gb1 if n_b1 else None,
                gw2 if n_w2 else None, gb2 if n_b2 else None, None, None, None, None)


def sdf_points(planes, w1, b1, w2, b2, points, scene_range, layout='channel_first', want_grad=True):
    d, g = SdfPoints.apply(planes, w1, b1, w2, b2, points, scene_range, layout, want_grad)
    return (d, g) if want_grad else (d, None)


def stratified_points(batch, nstrata, scene_range, device):
    """lib/ops.py:18-25 (same draw: ``torch.rand_like`` of a [B,n,n,n,3] tensor)."""
    n = nstrata - 1
    r = torch.arange(n, device=device)
    bins = torch.stack(torch.meshgrid(r, r, r, indexing='xy'), dim=-1).float()
    bins = bins.unsqueeze(0).expand(batch, -1, -1, -1, -1)
    bins = (bins + torch.rand_like(bins)) / n * 2 - 1
    return bins.flatten(1, 3) * scene_range


def laplace_cdf(x, beta):
    return 0.5 + 0.5 * torch.sign(x) * (1 - torch.exp(-x.abs() / beta))


def laplace_pdf(x, beta):
    return 0.5 * torch.exp(-x.abs() / beta) / beta


def regulariser_heads(planes, w1, b1, w2, b2, beta, scene_range, request, use_sdf=True,
                      training=True, layout='channel_first', nstrata=32):
    """generator.py:520-585 -> {'sdf_eikonal_loss': [B], ...} for the names in ``request``.
    ``planes`` [B,3,32,R,R] (or channel-last with ``layout``), EFFECTIVE decoder weights."""
    import torch.nn.functional as F
    out = {}
    wanted = [k for k in ('sdf_eikonal_loss', 'sdf_distance_loss', 'total_variation_loss',
                          'entropy_loss') if k in request]
    if not wanted:
        return out
    # (the reference enters the block only for eikonal / TV / entropy; a lone
    # 'sdf_distance_loss' request is never made by run.py: pre-training asks for both SDF terms)
    assert torch.is_grad_enabled()                      # generator.py:522
    B = planes.shape[0]
    pts = stratified_points(B, nstrata, scene_range, planes.device)
    eik = 'sdf_eikonal_loss' in request
    if eik:
        assert use_sdf and training                     # generator.py:531
    d, g = sdf_points(planes, w1, b1, w2, b2, pts, scene_range, layout, want_grad=eik)
    if eik:
        out['sdf_eikonal_loss'] = ((g.norm(dim=-1) - 1) ** 2).flatten(1).mean(dim=1)
    if 'sdf_distance_loss' in request:
        assert use_sdf
        with torch.no_grad():
            target = pts.norm(dim=-1) - 1               # unit sphere
        out['sdf_distance_loss'] = F.mse_loss(d.flatten(1), target.flatten(1),
                                              reduction='none').mean(dim=1)
    tv = 'total_variation_loss' in request
    if tv:
        coords = (pts / scene_range).view(B, 1, -1, 3)
        perturbed = coords + torch.randn_like(coords) * 0.004
        d2, _ = sdf_points(planes, w1, b1, w2, b2, perturbed.view(B, -1, 3) * scene_range,
                           scene_range, layout, want_grad=False)
    if use_sdf:
        if tv:
            out['total_variation_loss'] = F.l1_loss(laplace_cdf(-d, beta), laplace_cdf(-d2, beta),
                                                    reduction='none').flatten(1).mean(dim=1)
        if 'entropy_loss' in request:
            out['entropy_loss'] = laplace_pdf(-d, beta).flatten(1).mean(dim=1)
    else:
        t = torch.sigmoid(d - 1)
        if tv:
            out['total_variation_loss'] = F.l1_loss(t, torch.sigmoid(d2 - 1),
                                                    reduction='none').flatten(1).mean(dim=1)
        if 'entropy_loss' in request:
            out['entropy_loss'] = (t * (1 - t)).flatten(1).mean(dim=1)
    return out
