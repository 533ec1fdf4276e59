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

``__call__`` is forward only (evaluation renders, encoder-training targets, ``no_grad``
generator passes); a call that needs gradients raises.  The inversion setting -- every network
parameter frozen, gradients to the latents -- has its own entry:

    planes_cl = FusedSynthesis(net).forward_differentiable(ws, noise_mode='random')

which runs ``nfi_synthesis_forward_saved`` (the same planes, bit for bit, plus each layer's
pre-activation kept in the workspace) and, in backward, ``nfi_synthesis_backward`` to ws; a
network with a trainable parameter raises there.  The generator step -- gradients to ws and to
every parameter, noise strengths included -- has its own entry:

    planes_cl = FusedSynthesis(net).forward_trainable(ws, noise_mode='random')

backed by ``nfi_synthesis_backward_params``.  There is no CPU path and no fallback.
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
                 parameters=staticmethod(lambda: []))
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
        return self._run(ws, noise_mode, saved=False)[0]

    def forward_differentiable(self, ws, noise_mode='random'):
        """Channel-last planes [B,3,R,R,32] differentiable with respect to ``ws`` (every network
        parameter frozen).  The noise draws are the same draws, in the same order, as
        ``__call__``'s; the saved workspace lives until the backward has run."""
        assert noise_mode in ['random', 'const']
        if any(p.requires_grad for p in self.net.parameters()):
            raise _lib.NfiError(
                'FusedSynthesis.forward_differentiable differentiates to the latents only: every '
                'network parameter must be frozen (requires_grad_(False)); weight, bias and affine '
                'gradients are the reference module\'s')
        if not ws.is_cuda:
            raise _lib.NfiError('the fused synthesis network only runs on CUDA tensors '
                                '(there is no CPU path)')
        return _SynthesisFunction.apply(ws, self, noise_mode)

    def _layers(self):
        """(kind, block index, layer) of every layer with parameters, in the C ABI's order."""
        for i, blk in enumerate(self.blocks):
            if i:
                yield 'conv0', i, blk.conv0
            yield 'conv1', i, blk.conv1
            yield 'torgb', i, blk.torgb

    def forward_trainable(self, ws, noise_mode='random'):
        """Channel-last planes [B,3,R,R,32] differentiable with respect to ``ws`` and every
        network parameter (weights, biases, affines, ``b4.const``) -- the GAN generator step.  The
        per-layer noise tensors are formed here as ``raw * noise_strength`` (the same draws, in the
        same order, as ``__call__``'s) and enter the autograd Function as inputs, so autograd
        carries their gradient on to ``noise_strength``.  The backward runs
        ``nfi_synthesis_backward_params``; it is not differentiable (no ``create_graph``, so no
        path-length regulariser) and runs once per forward."""
        assert noise_mode in ['random', 'const']
        if not ws.is_cuda:
            raise _lib.NfiError('the fused synthesis network only runs on CUDA tensors '
                                '(there is no CPU path)')
        B, dev = ws.shape[0], ws.device
        noises = []   # per block (conv0, conv1), in the module's layer order like _run's draws
        for i, blk in enumerate(self.blocks):
            n0 = self._layer_noise(blk.conv0, B, noise_mode, dev) if i else None
            noises.append((n0, self._layer_noise(blk.conv1, B, noise_mode, dev)))
        params = []
        for _, _, layer in self._layers():
            params += [layer.weight, layer.affine.weight, layer.affine.bias, layer.bias]
        params.append(self.blocks[0].const)
        present = [(n0 is not None, n1 is not None) for n0, n1 in noises]
        flat_noise = [n for pair in noises for n in pair if n is not None]
        return _SynthesisTrainFunction.apply(ws, self, noise_mode, present, len(params),
                                             *params, *flat_noise)

    def _run(self, ws, noise_mode, saved, noises=None, trainable=False):
        """-> (planes, (P, keep, work)) -- P, keep and work stay valid for a backward.  ``noises``:
        per block (conv0, conv1) tensors drawn by the caller (else drawn here); ``trainable``
        sizes the workspace for the parameter backward."""
        net = self.net
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
                elif noises is not None:
                    fill(P.conv0[i], blk.conv0, noises[i][0])
                else:
                    fill(P.conv0[i], blk.conv0, self._layer_noise(blk.conv0, B, noise_mode, dev))
                if noises is not None:
                    fill(P.conv1[i], blk.conv1, noises[i][1])
                else:
                    fill(P.conv1[i], blk.conv1, self._layer_noise(blk.conv1, B, noise_mode, dev))
                fill(P.torgb[i], blk.torgb, None)
            P.ws = _ptr(ws)
            R = net.img_resolution
            planes = torch.empty(B, 3, R, R, 32, device=dev, dtype=torch.float32)
            P.planes = _ptr(planes)
            if trainable:
                sizer = lib.nfi_synthesis_param_workspace_bytes
            else:
                sizer = lib.nfi_synthesis_saved_workspace_bytes if saved else \
                    lib.nfi_synthesis_workspace_bytes
            need = sizer(ctypes.byref(P))
            if need == 0:
                raise _lib.NfiError('unsupported synthesis configuration (channels must be '
                                    'multiples of 32, resolution a power of two >= 8)')
            work = torch.empty(need, dtype=torch.uint8, device=dev)
            P.workspace, P.workspace_bytes = _ptr(work), need
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            fwd = lib.nfi_synthesis_forward_saved if saved else lib.nfi_synthesis_forward
            _lib.check(fwd(ctypes.byref(P), stream))
            # the launches are stream-ordered; `keep` / `work` may be released by the caching
            # allocator afterwards only for reuse on this same stream
        return planes, (P, keep, work)


class _SynthesisFunction(torch.autograd.Function):
    """ws -> planes (channel-last) with nfi_synthesis_backward as the backward."""

    @staticmethod
    def forward(ctx, ws, fs, noise_mode):
        planes, state = fs._run(ws, noise_mode, saved=True)
        ctx.state, ctx.ws_dtype = state, ws.dtype
        return planes

    @staticmethod
    def backward(ctx, g_planes):
        if ctx.state is None:
            raise _lib.NfiError('the fused synthesis backward ran twice on one forward '
                                '(retain_graph is not supported: the workspace is released)')
        if torch.is_grad_enabled():
            raise _lib.NfiError('the fused synthesis backward is not differentiable (create_graph, '
                                'e.g. the path-length regulariser): use the reference module')
        P, keep, work = ctx.state
        ctx.state = None          # the workspace and fp32 copies go once this returns
        dev = g_planes.device
        g_planes = g_planes.to(torch.float32).contiguous()
        ws32 = keep[0]
        g_ws = torch.zeros_like(ws32)
        G = _lib.SynthGrads(g_planes=g_planes.data_ptr(), g_ws=g_ws.data_ptr())
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.load().nfi_synthesis_backward(ctypes.byref(P), ctypes.byref(G), stream))
        del P, keep, work
        return g_ws.to(ctx.ws_dtype), None, None


class _SynthesisTrainFunction(torch.autograd.Function):
    """(ws, every parameter, the per-layer noise tensors) -> planes (channel-last), with
    nfi_synthesis_backward_params as the backward."""

    @staticmethod
    def forward(ctx, ws, fs, noise_mode, present, n_params, *tensors):
        params, flat_noise = tensors[:n_params], list(tensors[n_params:])
        noises = [(flat_noise.pop(0) if h0 else None, flat_noise.pop(0) if h1 else None)
                  for h0, h1 in present]
        planes, state = fs._run(ws, noise_mode, saved=True, noises=noises, trainable=True)
        ctx.state, ctx.fs, ctx.present, ctx.ws_dtype = state, fs, present, ws.dtype
        ctx.param_meta = [(p.shape, p.dtype) for p in params]
        ctx.noise_meta = [(n.shape, n.dtype) for pair in noises for n in pair if n is not None]
        return planes

    @staticmethod
    def backward(ctx, g_planes):
        if ctx.state is None:
            raise _lib.NfiError('the fused synthesis backward ran twice on one forward '
                                '(retain_graph is not supported: the workspace is released)')
        if torch.is_grad_enabled():
            raise _lib.NfiError('the fused synthesis backward is not differentiable (create_graph, '
                                'e.g. the path-length regulariser): use the reference module')
        P, keep, work = ctx.state
        ctx.state = None          # the workspace and fp32 copies go once this returns
        dev = g_planes.device
        g_planes = g_planes.to(torch.float32).contiguous()
        ws32 = keep[0]
        g_ws = torch.zeros_like(ws32)
        G = _lib.SynthGrads(g_planes=g_planes.data_ptr(), g_ws=g_ws.data_ptr())
        zeros = lambda shape: torch.zeros(shape, dtype=torch.float32, device=dev)
        g_params = [zeros(shape) for shape, _ in ctx.param_meta]
        g_noise = [zeros(shape) for shape, _ in ctx.noise_meta]
        PG = _lib.SynthParamGrads()
        k = 0
        for kind, i, _ in ctx.fs._layers():
            dst = getattr(PG, kind)[i]
            dst.g_weight, dst.g_affine_w, dst.g_affine_b, dst.g_bias = (
                _ptr(g) for g in g_params[k:k + 4])
            k += 4
        PG.g_const = _ptr(g_params[k])
        it = iter(g_noise)
        for i, (h0, h1) in enumerate(ctx.present):
            if h0:
                PG.conv0[i].g_noise = _ptr(next(it))
            if h1:
                PG.conv1[i].g_noise = _ptr(next(it))
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.load().nfi_synthesis_backward_params(
                ctypes.byref(P), ctypes.byref(G), ctypes.byref(PG), stream))
        del P, keep, work
        out = [g.to(dt) for g, (_, dt) in zip(g_params, ctx.param_meta)]
        out += [g.to(dt) for g, (_, dt) in zip(g_noise, ctx.noise_meta)]
        return (g_ws.to(ctx.ws_dtype), None, None, None, None, *out)


def planes_channel_first(planes_cl):
    """[B,3,R,R,32] -> the reference's [B,96,R,R] (tests, callers of the old layout)."""
    B, three, R, _, C = planes_cl.shape
    return planes_cl.permute(0, 1, 4, 2, 3).reshape(B, three * C, R, R)
