"""The tri-plane producer on sm_90a: ``SynthesisNetwork.forward`` behind the C ABI.

``FusedSynthesis(net)`` wraps the reference's UNMODIFIED ``models.stylegan.SynthesisNetwork``
(/root/reference/models/stylegan.py:438-490; it stays the owner of every parameter) and runs its
forward pass with the wgmma implicit-GEMM kernels of ``csrc/nfi_synth.cu`` through
``nfi_synthesis_forward`` (include/nfi_synth.h).  The call mirrors the module's:

    planes_cl = FusedSynthesis(net)(ws, noise_mode='random')     # [B,3,R,R,32] channel-last

i.e. what ``Generator.forward`` obtains at models/generator.py:475-477 as
``synthesis_network(w_synthesis, **block_kwargs).view(B,3,32,R,R)``, but already in the layout
``fused_render(..., planes_layout='channel_last')`` gathers from -- the 1.6 GB re-layout pass
between the two disappears.

Noise (stylegan.py:332-343): the per-layer ``torch.randn([B,1,res,res]) * noise_strength`` draws
are made HERE, in the module's layer order and from the same generator, so a seeded run consumes
the RNG like the reference; ``noise_mode='const'`` uses the registered ``noise_const`` buffers.

Forward only (evaluation renders, encoder-training targets, ``no_grad`` generator passes); a call
that needs gradients raises -- the inversion / GAN loops keep differentiating through the
reference module.  There is no CPU path and no fallback.
"""
import ctypes
import math

import torch

from . import _lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class _Layer:
    """Attribute view of one layer of a flat parameter dict (``from_params``)."""

    def __init__(self, p, prefix, resolution, use_noise, training):
        ns = lambda **kw: type('ns', (), kw)()
        self.weight, self.bias = p[prefix + '.weight'], p[prefix + '.bias']
        self.affine = ns(weight=p[prefix + '.affine.weight'], bias=p[prefix + '.affine.bias'])
        self.out_channels = self.weight.shape[0]
        self.resolution, self.training = resolution, training
        self.use_noise = use_noise and (prefix + '.noise_strength') in p
        if self.use_noise:
            self.noise_strength = p[prefix + '.noise_strength']
            self.noise_const = p[prefix + '.noise_const']


class FusedSynthesis:
    @classmethod
    def from_params(cls, p, training=False):
        """Builds the wrapper from the flat dict ``oracle.synthesis_oracle.extract_params``
        produces / the golden fixtures store (tensor names = the reference's state_dict keys,
        static facts under ``'meta'``) -- for callers that hold weights but not the module."""
        meta = p['meta']
        ns = lambda **kw: type('ns', (), kw)()
        net = ns(img_resolution=meta['img_resolution'], img_channels=meta['img_channels'],
                 w_dim=meta['w_dim'], block_resolutions=list(meta['resolutions']),
                 parameters=lambda: [])
        for r in meta['resolutions']:
            pre = 'b%d' % r
            blk = ns()
            for name in ('conv0', 'conv1'):
                key = '%s.%s' % (pre, name)
                if key in meta['layers']:
                    setattr(blk, name, _Layer(p, key, r, meta['layers'][key]['use_noise'], training))
            blk.torgb = _Layer(p, pre + '.torgb', r, False, training)
            if r == 4:
                blk.const = p[pre + '.const']
            setattr(net, pre, blk)
        return cls(net)

    def __init__(self, net):
        self.net = net
        self.resolutions = list(net.block_resolutions)
        self.blocks = [getattr(net, 'b%d' % r) for r in self.resolutions]
        if net.img_channels != 96:
            raise _lib.NfiError('the fused synthesis network emits 3 x 32-channel planes '
                                '(img_channels 96), got %d' % net.img_channels)
        if len(self.blocks) > _lib.SYNTH_MAX_BLOCKS:
            raise _lib.NfiError('img_resolution %d is beyond the %d blocks of the C ABI'
                                % (net.img_resolution, _lib.SYNTH_MAX_BLOCKS))

    # ------------------------------------------------------------------ noise, reference order
    def _layer_noise(self, layer, batch, noise_mode, device):
        """The tensor conv_modulated2d receives as ``noise`` (stylegan.py:332-343) or None."""
        if not layer.use_noise:
            return None
        if noise_mode == 'random' and (layer.training or bool(layer.noise_strength != 0)):
            n = torch.randn([batch, 1, layer.resolution, layer.resolution], device=device)
            return (n * layer.noise_strength).reshape(batch, layer.resolution, layer.resolution)
        if noise_mode == 'const' and bool(layer.noise_strength != 0):
            n = layer.noise_const * layer.noise_strength
            return n.unsqueeze(0).expand(batch, -1, -1)
        return None

    def __call__(self, ws, noise_mode='random'):
        assert noise_mode in ['random', 'const']  # stylegan.py:327
        net = self.net
        if torch.is_grad_enabled() and (ws.requires_grad or any(
                p.requires_grad for p in net.parameters())):
            raise _lib.NfiError(
                'FusedSynthesis is forward-only: call it under torch.no_grad() (or with frozen '
                'parameters and latents); differentiate through the reference module instead')
        if not ws.is_cuda:
            raise _lib.NfiError('the fused synthesis network only runs on CUDA tensors '
                                '(there is no CPU path)')
        lib = _lib.load()
        dev = ws.device
        B = ws.shape[0]
        ws = ws.detach().to(torch.float32).contiguous()
        assert ws.dim() == 3 and ws.shape[2] == net.w_dim, ws.shape
        P = _lib.SynthParams()
        P.batch, P.img_resolution, P.img_channels = B, net.img_resolution, net.img_channels
        P.w_dim, P.num_blocks, P.num_ws = net.w_dim, len(self.blocks), ws.shape[1]
        keep = [ws]

        def f32(t):
            t = t.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.to(torch.float32).contiguous()
            keep.append(t)
            return t

        def fill(dst, layer, noise):
            dst.weight = _ptr(f32(layer.weight))
            dst.affine_w = _ptr(f32(layer.affine.weight))
            dst.affine_b = _ptr(f32(layer.affine.bias))
            dst.bias = _ptr(f32(layer.bias))
            dst.noise = _ptr(f32(noise)) if noise is not None else None

        with torch.cuda.device(dev):
            for i, blk in enumerate(self.blocks):
                P.channels[i] = blk.conv1.out_channels
                if i == 0:
                    P.const_input = _ptr(f32(blk.const))
                else:
                    fill(P.conv0[i], blk.conv0, self._layer_noise(blk.conv0, B, noise_mode, dev))
                fill(P.conv1[i], blk.conv1, self._layer_noise(blk.conv1, B, noise_mode, dev))
                fill(P.torgb[i], blk.torgb, None)
            P.ws = _ptr(ws)
            R = net.img_resolution
            planes = torch.empty(B, 3, R, R, 32, device=dev, dtype=torch.float32)
            P.planes = _ptr(planes)
            need = lib.nfi_synthesis_workspace_bytes(ctypes.byref(P))
            if need == 0:
                raise _lib.NfiError('unsupported synthesis configuration (channels must be '
                                    'multiples of 32, resolution a power of two >= 8)')
            work = torch.empty(need, dtype=torch.uint8, device=dev)
            P.workspace, P.workspace_bytes = _ptr(work), need
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.nfi_synthesis_forward(ctypes.byref(P), stream))
            # the launches are stream-ordered; `keep` / `work` may be released by the caching
            # allocator afterwards only for reuse on this same stream
        return planes


def planes_channel_first(planes_cl):
    """[B,3,R,R,32] -> the reference's [B,96,R,R] (tests, callers of the old layout)."""
    B, three, R, _, C = planes_cl.shape
    return planes_cl.permute(0, 1, 4, 2, 3).reshape(B, three * C, R, R)
