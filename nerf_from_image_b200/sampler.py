"""The generator's ``sampler`` closure on the fused field kernel (seam B2).

``models/generator.py:587-681`` hands ``render`` a closure that evaluates the
radiance field at arbitrary points; besides ``render`` it serves point clouds
(iso-surface extraction, the regulariser grids, SDF pre-training targets).
``FusedSampler`` is the same callable -- same argument meaning, same output
names and shapes, same assertions -- backed by ``nfi_sample_field``:

    sampler = FusedSampler.from_generator(G, G(..., request_model_outputs=['sampler'])['sampler'])
    out = sampler(x_in, ['sigma', 'rgb'])        # x_in [B, ..., S, 3] world units

Forward only: the kernel does not record an autograd graph, so a call whose
inputs require grad while grad mode is on raises instead of silently returning
constants (the regulariser heads that differentiate through the closure keep
using the reference's own).  ``'normals'`` is the analytic gradient of the SDF
(the reference needs grad mode for its ``autograd.grad`` call; this one does
not).
"""

import ctypes

import torch

from . import _lib
from .fused import planes_to_channel_last

OUTPUT_NAMES = ('sdf_distance', 'sigma', 'rgb', 'normals', 'semantics', 'coords')


def _f32c(t, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.NfiError('%s must be a CUDA tensor: the fused sampler has no CPU path' % name)
    return t.detach().to(torch.float32).contiguous()


class FusedSampler:
    """Callable with the reference closure's signature (generator.py:587)."""

    def __init__(self, planes, w1, b1, w2, b2, palette, beta, alpha, scene_range,
                 use_sdf=True, bbox_debug=False, planes_channel_last=False):
        """planes [B,3,32,R,R] (or [B,3,R,R,32] with ``planes_channel_last``),
        EFFECTIVE decoder weights, palette [B,A,3] | None, beta/alpha [1]."""
        tensors = [planes, w1, b1, w2, b2, palette, beta, alpha]
        self._needs_grad = any(t is not None and t.requires_grad for t in tensors)
        planes = _f32c(planes, 'planes')
        self.planes_cl = planes if planes_channel_last else planes_to_channel_last(planes)
        self.w1, self.b1 = _f32c(w1, 'w1'), _f32c(b1, 'b1')
        self.w2, self.b2 = _f32c(w2, 'w2'), _f32c(b2, 'b2')
        self.palette = _f32c(palette, 'palette')
        self.beta = _f32c(beta, 'beta').reshape(1) if beta is not None else None
        self.alpha = _f32c(alpha, 'alpha').reshape(1) if alpha is not None else None
        self.scene_range = float(scene_range)
        self.use_sdf = bool(use_sdf)
        self.bbox_debug = bool(bbox_debug)
        self.attention_values = self.palette.shape[1] if self.palette is not None else 0
        n_out = 1 + (self.attention_values if self.attention_values > 0 else 3)
        if tuple(self.w2.shape) != (n_out, 64) or tuple(self.w1.shape) != (64, 32):
            raise _lib.NfiError('decoder weights must be [64,32] and [%d,64]' % n_out)
        if self.use_sdf and (self.beta is None or self.alpha is None):
            raise _lib.NfiError('use_sdf needs beta and alpha')

    @classmethod
    def from_generator(cls, target_model, sampler, scene_range=None, use_sdf=None,
                       bbox_debug=False):
        """Builds the fused sampler from a reference Generator and the closure
        (or ``model_outputs['triplane']`` dict) it returned."""
        from .render import extract_field
        planes, palette, w1, b1, w2, b2, beta, alpha = extract_field(target_model, sampler)
        if scene_range is None:
            scene_range = target_model.scene_range
        if use_sdf is None:
            use_sdf = bool(getattr(target_model, 'use_sdf', beta is not None))
        view_conditioned = bool(getattr(target_model, 'use_viewdir', False))
        if view_conditioned:
            # --use_viewdir: the decoder emits 1 + 32 values and the colour needs the per-RAY
            # view directions the reference closure captured (generator.py:242-251,662-663);
            # the seam serves the geometry outputs of such a model (row 0 of layer 2)
            n_col = palette.shape[1] if palette is not None else 3
            w2 = torch.cat((w2[:1], torch.zeros(n_col, 64, device=w2.device, dtype=w2.dtype)))
            b2 = torch.cat((b2[:1], torch.zeros(n_col, device=b2.device, dtype=b2.dtype)))
        out = cls(planes, w1, b1, w2, b2, palette, beta if use_sdf else None,
                  alpha if use_sdf else None, scene_range, use_sdf, bbox_debug)
        out.view_conditioned = view_conditioned
        return out

    def __call__(self, x_in, request_sampler_outputs=['sigma', 'rgb']):
        for output in request_sampler_outputs:
            assert output in OUTPUT_NAMES  # generator.py:588-592
        if 'normals' in request_sampler_outputs:
            assert self.use_sdf  # generator.py:600
        if 'semantics' in request_sampler_outputs:
            assert self.attention_values > 0  # generator.py:673
        if getattr(self, 'view_conditioned', False) and \
                ('rgb' in request_sampler_outputs or 'semantics' in request_sampler_outputs):
            raise NotImplementedError(
                "colours of a view-direction-conditioned model (--use_viewdir) need the rays' view "
                "directions: render() evaluates them; this seam offers 'sigma', 'sdf_distance', "
                "'normals' and 'coords' for such models")
        if torch.is_grad_enabled() and (self._needs_grad or x_in.requires_grad):
            raise _lib.NfiError(
                'the fused sampler is forward-only: call it under torch.no_grad(), or keep '
                "the reference's closure where gradients through the sampler are needed")
        bs = x_in.shape[0]
        if bs != self.planes_cl.shape[0]:
            raise _lib.NfiError('x_in batch %d != planes batch %d' % (bs, self.planes_cl.shape[0]))
        if x_in.shape[-1] != 3:
            raise _lib.NfiError('x_in must end in 3 coordinates')
        pts = _f32c(x_in, 'x_in').reshape(bs, -1, 3)
        n = pts.shape[1]
        dev = pts.device
        new = lambda *shape: torch.empty(shape, device=dev, dtype=torch.float32)
        want = set(request_sampler_outputs)
        bufs = dict(
            sdf_distance=new(bs, n, 1) if 'sdf_distance' in want else None,
            sigma=new(bs, n) if 'sigma' in want else None,
            rgb=new(bs, n, 3) if 'rgb' in want else None,
            semantics=new(bs, n, self.attention_values) if 'semantics' in want else None,
            normals=new(bs, n, 3) if 'normals' in want else None)
        out = {}
        if any(b is not None for b in bufs.values()):
            if self.bbox_debug and bufs['sigma'] is None:
                raise _lib.NfiError("bbox_debug adds to 'sigma': request it")
            sp = _lib.SampleParams()
            sp.batch, sp.plane_res = bs, self.planes_cl.shape[2]
            sp.n_attention, sp.use_sdf = self.attention_values, int(self.use_sdf)
            # generator.py:640: the debug box is only drawn when 'coords' is requested too
            sp.bbox_debug = int(self.bbox_debug and 'coords' in want)
            sp.scene_range, sp.n_points = self.scene_range, n
            for k, t in (('planes', self.planes_cl), ('w1', self.w1), ('b1', self.b1),
                         ('w2', self.w2), ('b2', self.b2), ('palette', self.palette),
                         ('beta', self.beta), ('alpha', self.alpha), ('points', pts)):
                setattr(sp, k, _lib.ptr(t))
            for k, t in bufs.items():
                setattr(sp, k, _lib.ptr(t))
            lib = _lib.load()
            with torch.cuda.device(dev):
                _lib.check(lib.nfi_sample_field(ctypes.byref(sp), _lib.stream(dev)))
        for k, t in bufs.items():
            if t is not None:
                out[k] = t
        if 'normals' in out:  # the reference returns them in x_in's shape (generator.py:619)
            out['normals'] = out['normals'].reshape(x_in.shape)
        if 'coords' in want:
            out['coords'] = x_in
        return out
