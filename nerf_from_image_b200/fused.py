"""torch.autograd.Function over the C ABI of libnfi_render.so.

``FusedTriplaneRender.apply`` is the differentiable core that
``nerf_from_image_b200.render.render`` (the drop-in for
/root/reference/run.py:176-350) calls once the planes and palette have been
produced by the generator front-end.  Tensors stay torch tensors (device
memory, streams); all arithmetic of the path happens in the CUDA library.
"""

import ctypes
from dataclasses import dataclass

import torch

from . import _lib
from .rays import unit_rays


@dataclass(frozen=True)
class RenderConfig:
    """What render() reads from the reference's module globals
    (run.py:200,216,229,232,259,348: args.* and dataset_config[*])."""
    scene_range: float
    white_background: bool = False
    use_sdf: bool = True
    fine_sampling: bool = True
    attention_values: int = 10
    mlp_mode: int = _lib.MLP_AUTO


# bench.py sets this to a list to collect (start, end) CUDA events around the
# render kernel launch (events on the launching stream); None = no timing.
KERNEL_EVENTS = None
# timing experiments: a float32 CUDA tensor of >= 16 elements the kernel fills with
# per-phase cycle counts when mlp_mode has bit 0x1000 set
DEBUG_BUF = None
# backward trace of one ray (tools/grad_trace.py): ray index b*H*W + y*W + x, or None
DEBUG_RAY = None


def _f32c(t, name):
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError('%s must be float32 (the reference path is strict '
                        'fp32, run.py:59-60), got %s' % (name, t.dtype))
    return t.contiguous()


def planes_to_channel_last(planes):
    """[B,3,32,R,R] (views of the synthesis output) -> [B,3,R,R,32]."""
    B, three, C, R, R2 = planes.shape
    assert three == 3 and C == 32 and R == R2, planes.shape
    planes = _f32c(planes, 'planes')
    out = torch.empty(B, 3, R, R, C, device=planes.device, dtype=torch.float32)
    lib = _lib.load()
    stream = _lib.stream(planes.device)
    base = planes.data_ptr()
    step = C * R * R * 4
    _lib.check(lib.nfi_planes_to_channel_last(
        ctypes.c_void_p(base), ctypes.c_void_p(base + step),
        ctypes.c_void_p(base + 2 * step), 3 * C * R * R, B, R, _lib.ptr(out), stream))
    return out


def planes_from_channel_last(planes_cl):
    B, three, R, R2, C = planes_cl.shape
    out = torch.empty(B, 3, C, R, R, device=planes_cl.device, dtype=torch.float32)
    lib = _lib.load()
    stream = _lib.stream(planes_cl.device)
    _lib.check(lib.nfi_planes_from_channel_last(_lib.ptr(planes_cl), B, R, _lib.ptr(out), stream))
    return out


def _make_params(cfg, planes_cl, w1, b1, w2, b2, palette, beta, alpha, c2w,
                 focal, center, bbox, height, width, S, noise_t, noise_u,
                 extra_mode, view_feat=None, w3=None, b3=None, rows=None):
    p = _lib.RenderParams()
    B, _, R, _, _ = planes_cl.shape
    p.batch, p.height, p.width, p.num_samples = B, height, width, S
    p.plane_res = R
    p.n_attention = cfg.attention_values
    p.scene_range = cfg.scene_range
    p.white_background = int(cfg.white_background)
    p.use_sdf = int(cfg.use_sdf)
    p.fine_sampling = int(cfg.fine_sampling)
    p.noise_mode = _lib.NOISE_EXPLICIT if noise_t is not None else _lib.NOISE_DETERMINISTIC
    p.extra_mode = extra_mode
    p.compute_normals = 0
    p.mlp_mode = cfg.mlp_mode
    p.planes, p.w1, p.b1, p.w2, p.b2 = (_lib.ptr(planes_cl), _lib.ptr(w1), _lib.ptr(b1),
                                        _lib.ptr(w2), _lib.ptr(b2))
    p.palette, p.beta, p.alpha = _lib.ptr(palette), _lib.ptr(beta), _lib.ptr(alpha)
    p.c2w, p.focal, p.center, p.bbox = _lib.ptr(c2w), _lib.ptr(focal), _lib.ptr(center), _lib.ptr(bbox)
    p.noise_t, p.noise_u = _lib.ptr(noise_t), _lib.ptr(noise_u)
    p.view_features, p.w3, p.b3 = _lib.ptr(view_feat), _lib.ptr(w3), _lib.ptr(b3)
    if rows is not None:
        p.row_offset, p.full_height = int(rows[0]), int(rows[1])
    return p


def _check_shapes(cfg, planes, w1, b1, w2, b2, palette, c2w, focal, center,
                  bbox, height, width, S, noise_t, noise_u, channel_last=False,
                  view_feat=None, w3=None, b3=None):
    B = planes.shape[0]
    A = cfg.attention_values
    nout = 1 + (A if A > 0 else 3)
    if view_feat is not None:
        # --use_viewdir: the decoder emits 1 + 32 values, the colour logits come from the
        # mapper's output layer (generator.py:376-377,395-396)
        assert tuple(view_feat.shape) == (B, height, width, 32), view_feat.shape
        assert w3 is not None and tuple(w3.shape) == (nout - 1, 32), (None if w3 is None else w3.shape)
        assert b3 is not None and tuple(b3.shape) == (nout - 1,)
        nout = 33
    if channel_last:
        assert (planes.dim() == 5 and planes.shape[1] == 3 and planes.shape[4] == 32
                and planes.shape[2] == planes.shape[3]), planes.shape
    else:
        assert planes.dim() == 5 and planes.shape[1:3] == (3, 32), planes.shape
    assert tuple(w1.shape) == (64, 32) and tuple(b1.shape) == (64,)
    assert tuple(w2.shape) == (nout, 64) and tuple(b2.shape) == (nout,), \
        (w2.shape, nout)
    if A > 0:
        assert palette is not None and tuple(palette.shape) == (B, A, 3), \
            (None if palette is None else palette.shape)
    assert tuple(c2w.shape) == (B, 4, 4), c2w.shape
    assert focal is None or tuple(focal.shape) == (B,), focal.shape
    assert center is None or tuple(center.shape) == (B, 2)
    assert bbox is None or tuple(bbox.shape) == (B, 2, 2)
    if noise_t is not None:
        assert tuple(noise_t.shape) == (B, height, width, S), noise_t.shape
        if cfg.fine_sampling:
            assert noise_u is not None and tuple(noise_u.shape) == (B * height * width, S)
    for t in (planes, w1, b1, w2, b2, palette, c2w, focal, center, bbox, noise_t, noise_u,
              view_feat, w3, b3):
        if t is not None and not t.is_cuda:
            raise _lib.NfiError('the fused renderer only runs on CUDA tensors '
                                '(there is no CPU path)')


_FIELD_KEYS = ('w1', 'b1', 'w2', 'b2', 'palette', 'beta', 'alpha', 'c2w', 'focal', 'center',
               'bbox', 'noise_t', 'noise_u', 'view_feat', 'w3', 'b3')


class FusedTriplaneRender(torch.autograd.Function):
    """(planes, decoder, palette, beta, alpha, cameras) -> (rgb, depth, mask, extra).

    planes [B,3,32,R,R]; w1 [64,32], b1 [64], w2 [1+A,64], b2 [1+A] are the
    EFFECTIVE decoder weights; palette [B,A,3]; beta, alpha [1]; c2w [B,4,4];
    focal [B]|None; center [B,2]|None; bbox [B,2,2]|None.  ``noise_t`` /
    ``noise_u`` None selects the reference's ``randomize=False`` behaviour.
    ``extra_mode``: 0 none, 1 coords, 2 semantics.  ``cam_grad`` False is the
    reference's ``force_no_cam_grad``.  ``view_feat`` [B,H,W,32] / ``w3`` [A,32] / ``b3`` [A]:
    the ViewDirectionMapper's per-ray trunk output and its output layer (--use_viewdir,
    generator.py:189-253); w2 / b2 then have 33 rows.
    """

    @staticmethod
    def forward(ctx, planes, w1, b1, w2, b2, palette, beta, alpha, c2w, focal,
                center, bbox, cfg, height, width, S, noise_t, noise_u,
                extra_mode, cam_grad, compute_normals=False, out=None,
                planes_layout='channel_first', peers=None, view_feat=None, w3=None, b3=None,
                rows=None):
        channel_last = planes_layout == 'channel_last'
        _check_shapes(cfg, planes, w1, b1, w2, b2, palette, c2w, focal, center,
                      bbox, height, width, S, noise_t, noise_u, channel_last, view_feat, w3, b3)
        lib = _lib.load()
        dev = planes.device
        with torch.cuda.device(dev):
            stream = _lib.stream(dev)
            # [B,3,R,R,32] as synthesis.FusedSynthesis emits it: no re-layout pass
            planes_cl = (_f32c(planes.detach(), 'planes') if channel_last
                         else planes_to_channel_last(planes.detach()))
            t = dict(w1=_f32c(w1.detach(), 'w1'), b1=_f32c(b1.detach(), 'b1'),
                     w2=_f32c(w2.detach(), 'w2'), b2=_f32c(b2.detach(), 'b2'),
                     palette=_f32c(palette.detach(), 'palette') if palette is not None else None,
                     beta=_f32c(beta.detach(), 'beta') if cfg.use_sdf else None,
                     alpha=_f32c(alpha.detach(), 'alpha') if cfg.use_sdf else None,
                     c2w=_f32c(c2w.detach(), 'tform_cam2world'),
                     focal=_f32c(focal.detach(), 'focal_length') if focal is not None else None,
                     center=_f32c(center.detach(), 'center') if center is not None else None,
                     bbox=_f32c(bbox.detach(), 'bbox') if bbox is not None else None,
                     noise_t=_f32c(noise_t, 'noise_t'), noise_u=_f32c(noise_u, 'noise_u'),
                     view_feat=_f32c(view_feat.detach(), 'view_feat') if view_feat is not None else None,
                     w3=_f32c(w3.detach(), 'w3') if view_feat is not None else None,
                     b3=_f32c(b3.detach(), 'b3') if view_feat is not None else None)
            B = planes.shape[0]
            A = cfg.attention_values
            needs_grad = any(ctx.needs_input_grad)
            if out is not None:
                # caller-owned outputs (parallel.render_sharded: this rank's slices of the
                # all-gathered buffers, so that the collective runs in place)
                rgb, depth, mask = out
                for o, shape in ((rgb, (B, height, width, 3)), (depth, (B, height, width)),
                                 (mask, (B, height, width))):
                    if (tuple(o.shape) != shape or o.dtype != torch.float32
                            or o.device != dev or not o.is_contiguous()):
                        raise _lib.NfiError('out= must be contiguous fp32 CUDA tensors of shapes '
                                            '[B,H,W,3], [B,H,W], [B,H,W] on the planes\' device')
            else:
                rgb = torch.empty(B, height, width, 3, device=dev)
                depth = torch.empty(B, height, width, device=dev)
                mask = torch.empty(B, height, width, device=dev)
            extra = None
            if extra_mode == _lib.EXTRA_COORDS:
                extra = torch.empty(B, height, width, 3, device=dev)
            elif extra_mode == _lib.EXTRA_SEMANTICS:
                extra = torch.empty(B, height, width, A, device=dev)
            normals = None
            if compute_normals:
                # models/generator.py:599-601: SDF models only; forward quantity, no gradient
                # (create_graph=False, weights detached: lib/nerf_utils.py:146-148)
                assert cfg.use_sdf
                normals = torch.empty(B, height, width, 3, device=dev)
            z_fine = None
            if (needs_grad or compute_normals) and cfg.fine_sampling:
                # the fine depths: kept for the backward pass, and read by the normals kernel
                z_fine = torch.empty(B * height * width, S, device=dev)
            p = _make_params(cfg, planes_cl, t['w1'], t['b1'], t['w2'], t['b2'],
                             t['palette'], t['beta'], t['alpha'], t['c2w'],
                             t['focal'], t['center'], t['bbox'], height, width,
                             S, t['noise_t'], t['noise_u'], extra_mode,
                             t['view_feat'], t['w3'], t['b3'], rows)
            p.rgb, p.depth, p.mask = _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(mask)
            p.extra = _lib.ptr(extra)
            p.z_fine = _lib.ptr(z_fine)
            if normals is not None:
                p.compute_normals, p.normals = 1, _lib.ptr(normals)
            if DEBUG_BUF is not None:
                p.normals = _lib.ptr(DEBUG_BUF)
            if peers:
                # raw device addresses of this rank's [rgb, depth, mask] slices inside each peer's
                # buffers (parallel.PeerExchange): the kernel stores its tiles there as well
                if len(peers['slices'] if isinstance(peers, dict) else peers) > _lib.MAX_PEERS:
                    raise _lib.NfiError('at most %d peers' % _lib.MAX_PEERS)
                slices = peers['slices'] if isinstance(peers, dict) else peers
                p.n_peers = len(slices)
                for q, (pr, pd, pm) in enumerate(slices):
                    p.peer_rgb[q], p.peer_depth[q], p.peer_mask[q] = int(pr), int(pd), int(pm)
                if isinstance(peers, dict) and peers.get('done') is not None:
                    # completion handshake inside the kernel (parallel.PeerExchange)
                    for q, (sig, r) in enumerate(zip(peers['signal'], peers['ranks'])):
                        p.peer_signal[q], p.peer_rank[q] = int(sig), int(r)
                    p.peer_signal_self = int(peers['self_signal'])
                    p.peer_epoch = int(peers['epoch']) & 0xFFFFFFFF
                    p.peer_done = int(peers['done'])
            ws_bytes = lib.nfi_render_workspace_bytes(ctypes.byref(p))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            p.workspace, p.workspace_bytes = _lib.ptr(ws), ws_bytes
            if KERNEL_EVENTS is not None:
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                e0.record()
            _lib.check(lib.nfi_render_forward(ctypes.byref(p), stream))
            if KERNEL_EVENTS is not None:
                e1.record()
                KERNEL_EVENTS.append((e0, e1))
        if needs_grad:
            # Only non-tensor configuration lives on ctx.  Every tensor goes through
            # save_for_backward: no output -> grad_fn -> ctx -> output cycle (the buffers are
            # released with the graph, not by the cyclic GC), and an in-place edit of a
            # returned output before backward() trips autograd's version check instead of
            # silently corrupting the total L that backward rebuilds from rgb / mask / extra.
            ctx.cfg, ctx.dims, ctx.extra_mode = cfg, (height, width, S), extra_mode
            ctx.cam_grad = cam_grad
            ctx.channel_last = channel_last
            ctx.rows = rows
            # caller-owned outputs are slices of buffers an in-place all-gather completes
            # afterwards (parallel.py); it rewrites this rank's slice with the values it
            # already holds, so those are saved as aliases with their own version counter
            keep = (lambda x: x) if out is None else (lambda x: x.data)
            saved = dict(t, out_rgb=keep(rgb), out_mask=keep(mask), out_extra=extra,
                         planes_cl=planes_cl, z_fine=z_fine)
            ctx.saved_names = [k for k, v in saved.items() if v is not None]
            ctx.save_for_backward(*[saved[k] for k in ctx.saved_names])
        ctx.mark_non_differentiable(depth)
        if extra is None:
            extra = torch.empty(0, device=dev)
            ctx.mark_non_differentiable(extra)
        if normals is None:
            normals = torch.empty(0, device=dev)
        ctx.mark_non_differentiable(normals)
        return rgb, depth, mask, extra, normals

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_mask, g_extra, g_normals=None):
        cfg, (height, width, S) = ctx.cfg, ctx.dims
        lib = _lib.load()
        saved = dict(zip(ctx.saved_names, ctx.saved_tensors))
        t = {k: saved.get(k) for k in _FIELD_KEYS}
        planes_cl, z_fine = saved['planes_cl'], saved.get('z_fine')
        dev = planes_cl.device
        need = ctx.needs_input_grad
        (n_planes, n_w1, n_b1, n_w2, n_b2, n_pal, n_beta, n_alpha, n_c2w,
         n_focal, n_center, n_bbox) = need[:12]
        n_vf, n_w3, n_b3 = need[24:27]
        rgb, mask, extra = saved['out_rgb'], saved['out_mask'], saved.get('out_extra')
        A = cfg.attention_values
        with torch.cuda.device(dev):
            stream = _lib.stream(dev)
            z = lambda ref: torch.zeros_like(ref)
            g = _lib.RenderGrads()
            g_rgb = _f32c(g_rgb, 'grad rgb') if g_rgb is not None else torch.zeros_like(rgb)
            g.g_rgb = _lib.ptr(g_rgb)
            g_mask = _f32c(g_mask, 'grad mask') if g_mask is not None else None
            g.g_mask = _lib.ptr(g_mask)
            if extra is not None and g_extra is not None and g_extra.numel() > 0:
                g_extra = _f32c(g_extra, 'grad extra')
                g.g_extra, g.out_extra = _lib.ptr(g_extra), _lib.ptr(extra)
            g.out_rgb, g.out_mask = _lib.ptr(rgb), _lib.ptr(mask)
            gp_cl = z(planes_cl) if n_planes else None
            gw1 = z(t['w1']) if n_w1 else None
            gb1 = z(t['b1']) if n_b1 else None
            gw2 = z(t['w2']) if n_w2 else None
            gb2 = z(t['b2']) if n_b2 else None
            gpal = z(t['palette']) if (n_pal and A > 0) else None
            gbeta = z(t['beta']) if (n_beta and cfg.use_sdf) else None
            galpha = z(t['alpha']) if (n_alpha and cfg.use_sdf) else None
            cam = ctx.cam_grad and (n_c2w or n_focal or n_center or n_bbox)
            go = torch.zeros(rgb.shape, device=dev) if cam else None
            gd = torch.zeros(rgb.shape, device=dev) if cam else None
            vd = t['view_feat'] is not None
            gvf = z(t['view_feat']) if (vd and n_vf) else None
            gw3 = z(t['w3']) if (vd and n_w3) else None
            gb3 = z(t['b3']) if (vd and n_b3) else None
            g.grad_view_features, g.grad_w3, g.grad_b3 = _lib.ptr(gvf), _lib.ptr(gw3), _lib.ptr(gb3)
            (g.grad_planes, g.grad_w1, g.grad_b1, g.grad_w2, g.grad_b2,
             g.grad_palette, g.grad_beta, g.grad_alpha, g.grad_origins,
             g.grad_dirs) = (_lib.ptr(gp_cl), _lib.ptr(gw1), _lib.ptr(gb1), _lib.ptr(gw2),
                             _lib.ptr(gb2), _lib.ptr(gpal), _lib.ptr(gbeta), _lib.ptr(galpha),
                             _lib.ptr(go), _lib.ptr(gd))
            p = _make_params(cfg, planes_cl, t['w1'], t['b1'], t['w2'], t['b2'],
                             t['palette'], t['beta'], t['alpha'], t['c2w'],
                             t['focal'], t['center'], t['bbox'], height, width,
                             S, t['noise_t'], t['noise_u'], ctx.extra_mode,
                             t['view_feat'], t['w3'], t['b3'], ctx.rows)
            p.rgb, p.depth, p.mask = _lib.ptr(rgb), _lib.ptr(mask), _lib.ptr(mask)  # unused
            p.extra = _lib.ptr(extra)
            p.z_fine = _lib.ptr(z_fine)
            if DEBUG_RAY is not None and DEBUG_BUF is not None:
                p.normals, p.noise_seed = _lib.ptr(DEBUG_BUF), int(DEBUG_RAY)
                p.mlp_mode = cfg.mlp_mode | 0x4000
            # the tensor-core backward keeps its two weight images here (64 KiB; 96 KiB for a
            # view-conditioned decoder, whose weight gradients stay on the SIMT kernel), the
            # weight-gradient kernel one accumulator row buffer per CTA behind them
            if vd:
                ws_bytes = _lib.VIEW_BACKWARD_WORKSPACE_BYTES
            else:
                ws_bytes = (_lib.BACKWARD_WORKSPACE_BYTES if (n_w1 or n_b1 or n_w2 or n_b2)
                            else _lib.BACKWARD_IMAGES_BYTES)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            p.workspace, p.workspace_bytes = _lib.ptr(ws), ws_bytes
            _lib.check(lib.nfi_render_backward(ctypes.byref(p), ctypes.byref(g), stream))
            gplanes = None
            if n_planes:  # gradient in the layout the planes came in
                gplanes = gp_cl if ctx.channel_last else planes_from_channel_last(gp_cl)
            gc2w = gfocal = gcenter = gbbox = None
            if cam:
                # chain (dL/d origin, dL/d unit dir) to the camera parameters
                with torch.enable_grad():
                    leaf = lambda x, n: (x.detach().requires_grad_(True)
                                         if (x is not None and n) else x)
                    c2w_l = leaf(t['c2w'], n_c2w)
                    focal_l = leaf(t['focal'], n_focal)
                    center_l = leaf(t['center'], n_center)
                    bbox_l = leaf(t['bbox'], n_bbox)
                    o, d = unit_rays(height, width, c2w_l, focal_l, center_l, bbox_l, ctx.rows)
                    leaves = [x for x, n in ((c2w_l, n_c2w), (focal_l, n_focal),
                                             (center_l, n_center), (bbox_l, n_bbox))
                              if x is not None and n]
                    # an orthographic camera with only bbox requiring grad moves the origins
                    # but not the directions (and the perspective case the reverse)
                    pairs = [(x, gx) for x, gx in ((o, go), (d, gd)) if x.requires_grad]
                    outs = [x for x, _ in pairs]
                    gos = [gx for _, gx in pairs]
                    res = list(torch.autograd.grad(outs, leaves, gos, allow_unused=True))
                if t['c2w'] is not None and n_c2w:
                    gc2w = res.pop(0)
                if t['focal'] is not None and n_focal:
                    gfocal = res.pop(0)
                if t['center'] is not None and n_center:
                    gcenter = res.pop(0)
                if t['bbox'] is not None and n_bbox:
                    gbbox = res.pop(0)
        return (gplanes, gw1, gb1, gw2, gb2, gpal, gbeta, galpha, gc2w, gfocal,
                gcenter, gbbox, None, None, None, None, None, None, None, None, None, None,
                None, None, gvf, gw3, gb3, None)


def fused_render(planes, w1, b1, w2, b2, palette, beta, alpha, c2w, focal,
                 center, bbox, cfg, height, width, num_samples, noise_t=None,
                 noise_u=None, extra_mode=_lib.EXTRA_NONE, cam_grad=True,
                 compute_normals=False, out=None, planes_layout='channel_first', peers=None,
                 view=None, rows=None):
    """Functional form; returns (rgb, depth, mask, extra|None), with
    ``compute_normals`` (rgb, depth, mask, extra|None, normals).  ``out=(rgb, depth,
    mask)`` makes the kernel write into caller-owned tensors (see parallel.py).
    ``planes_layout``: 'channel_first' = [B,3,32,R,R] as the reference's synthesis network
    leaves them (re-laid-out here), 'channel_last' = [B,3,R,R,32] as synthesis.FusedSynthesis
    emits them (used as they are; a plane gradient comes back in the same layout).
    ``peers``: list of (rgb, depth, mask) device ADDRESSES of this rank's slices in the other
    ranks' buffers; the kernel stores its tiles there too (parallel.PeerExchange).
    ``view``: (view_features [B,H,W,32], w3 [A,32], b3 [A]) switches on the view-direction
    conditioning of the CARLA models (--use_viewdir; the forward, and the backward with frozen
    decoder and mapper output, on the pipelined tensor-core kernels where they can take the
    configuration, the GAN step's decoder / mapper-output gradients on the fp32 SIMT kernel).
    ``rows``: (row_offset, full_height) renders rows [row_offset, row_offset + height) of images
    full_height rows tall; every per-ray tensor (noise, outputs) then has ``height`` rows.

    The kernels compute in fp32 like the reference's render (run.py:59-60).  Under
    autocast (BASELINE config 4 trains the synthesis network in bf16) the field tensors
    may arrive in half precision: they are widened here, differentiably, so the
    gradients flow back in the caller's dtype."""
    def f32(t):
        return t.float() if (t is not None and t.dtype in (torch.float16, torch.bfloat16)) else t
    planes, w1, b1, w2, b2, palette, beta, alpha = map(f32, (planes, w1, b1, w2, b2, palette,
                                                              beta, alpha))
    c2w, focal, center, bbox = map(f32, (c2w, focal, center, bbox))
    view_feat, w3, b3 = map(f32, view) if view is not None else (None, None, None)
    rgb, depth, mask, extra, normals = FusedTriplaneRender.apply(
        planes, w1, b1, w2, b2, palette, beta, alpha, c2w, focal, center, bbox,
        cfg, height, width, num_samples, noise_t, noise_u, extra_mode, cam_grad,
        compute_normals, out, planes_layout, peers, view_feat, w3, b3, rows)
    extra = extra if extra_mode != _lib.EXTRA_NONE else None
    if compute_normals:
        return rgb, depth, mask, extra, normals
    return rgb, depth, mask, extra
