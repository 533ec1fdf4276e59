"""The GAN discriminator's backbone on sm_90a (``include/nfi_disc.h``).

Every GAN iteration calls the reference's ``Discriminator`` (models/discriminator.py) several times:
``D(rendered image)`` in the generator step (D frozen, gradient to the image), ``D(real)`` and
``D(fake)`` in the discriminator step (gradients to every D parameter), and on every other D step
the R1 call, whose real-image gradient is differentiated again.  ``enable_fused_discriminator``
switches a reference ``Discriminator`` instance to a forward with the same contract:

- the conditioning vector (``matrix_to_conditioning_vector``) and the two-layer conditioning mapping
  network run as they are, in torch; the map ``cmap`` they produce enters the kernels, and its
  gradient comes back so that autograd carries it on through the mapping;
- from the image and ``cmap`` to the logits, one autograd function runs ``nfi_disc_forward`` and,
  in its backward, ``nfi_disc_backward``: gradients to the image, ``cmap`` and every backbone weight
  and bias;
- the R1 call runs the module's own ``forward``.  It is recognisable at call time: the image
  requires grad AND some weight or bias of the module does (read by attribute, so that an
  ``nn.DataParallel`` replica, which registers no parameters, is judged alike).  In the generator
  step the parameters are
  frozen, and in the discriminator step's other calls the image does not require grad.  So R1's
  penalty and its gradients are the module's -- unless ``enable_fused_discriminator(D, r1=True)``:
  then the R1 call runs ``nfi_disc_forward`` too, its create_graph backward returns the gradients
  through a second autograd function (forward ``nfi_disc_backward``, backward
  ``nfi_disc_backward_hvp``, include/nfi_disc_r1.h), and its plain backward is the first-order one.
  One saved forward serves those three passes and is released when no pass can still come.

The binding is one line after each discriminator is built, before ``nn.DataParallel``::

    enable_fused_discriminator(discriminator)

The instance's class is swapped for a subclass that overrides ``forward``, so ``nn.DataParallel``'s
replicas run the fused forward too, and the parameters, their names and ``state_dict()`` are the
module's own.  Calls outside the kernels' envelope (an image encoder or class embedding as
condition, a batch that is not a multiple of 4, a resolution outside 8..256 or a layout other than
the reference's) run the module's forward.  Refused with ``NfiError``: CPU or non-fp32 tensors, a
double backward (``create_graph``) and a second backward of one forward; for the R1 call, a second
create_graph backward, a third backward, a third derivative and a cotangent on its ``cmap`` or
parameter gradients.
"""
import ctypes
import math
import sys

import torch

from . import _lib

C4 = 512
MAX_BLOCKS = _lib.DISC_MAX_BLOCKS


def channels(r):
    return min(32768 // r, C4)


def block_resolutions(R):
    return [R >> i for i in range(int(math.log2(R)) - 2)]


def _layout_ok(bb):
    """Whether a DiscriminatorBackbone-shaped module ``bb`` is laid out as stylegan.py:609-662 with
    the defaults run.py uses."""
    try:
        R, nc = bb.img_resolution, bb.img_channels
        if not (8 <= R <= 256 and R & (R - 1) == 0 and 1 <= nc <= 4):
            return False
        if list(bb.block_resolutions) != block_resolutions(R):
            return False
        for i, r in enumerate(block_resolutions(R)):
            blk = getattr(bb, 'b%d' % r)
            c, co = channels(r), channels(r // 2)
            if blk.conv0.weight.shape != (c, c, 3, 3) or blk.conv1.weight.shape != (co, c, 3, 3):
                return False
            if blk.skip.weight.shape != (co, c, 1, 1) or blk.skip.bias is not None:
                return False
            if (i == 0) != hasattr(blk, 'fromrgb'):
                return False
            if i == 0 and blk.fromrgb.weight.shape != (c, nc, 1, 1):
                return False
        b4 = bb.b4
        if b4.mbstd is None or b4.mbstd.group_size != 4 or b4.mbstd.num_channels != 1:
            return False
        if b4.conv.weight.shape != (C4, C4 + 1, 3, 3) or b4.fc.weight.shape != (C4, 16 * C4):
            return False
        if b4.cmap_dim not in (0, C4) or b4.out.weight.shape[1] != C4:
            return False
        return bb.c_dim >= 0 and (bb.c_dim == 0) == (b4.cmap_dim == 0)
    except AttributeError:
        return False


def parameters_of(bb):
    """The backbone's weights and biases in the order the kernels take them: fromrgb (w, b); per
    block conv0 (w, b), conv1 (w, b), skip w; b4.conv (w, b), b4.fc (w, b), b4.out (w, b)."""
    R = bb.img_resolution
    rs = block_resolutions(R)
    first = getattr(bb, 'b%d' % R).fromrgb
    ps = [first.weight, first.bias]
    for r in rs:
        blk = getattr(bb, 'b%d' % r)
        ps += [blk.conv0.weight, blk.conv0.bias, blk.conv1.weight, blk.conv1.bias, blk.skip.weight]
    b4 = bb.b4
    return ps + [b4.conv.weight, b4.conv.bias, b4.fc.weight, b4.fc.bias, b4.out.weight, b4.out.bias]


def logits(bb, img, cmap, r1=False):
    """The backbone's output [B,1] from the image [B,nc,R,R] and the conditioning map [B,512] (None
    for an unconditional backbone), on the kernels.  ``r1``: the call's image gradient may be
    differentiated again (``_DiscR1Function``)."""
    ps = parameters_of(bb)
    if r1:
        return _DiscR1Function.apply(img, cmap, *ps)
    needs = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in [img, cmap] + ps)
    return _DiscFunction.apply(int(needs), img, cmap, *ps)


def _params(img, cmap, ws, save):
    B, nc, R = img.shape[0], img.shape[1], img.shape[2]
    nb = len(block_resolutions(R))
    p = _lib.DiscParams()
    p.batch, p.resolution, p.img_channels = B, R, nc
    p.cmap_dim, p.save = (cmap.shape[1] if cmap is not None else 0), save
    p.img, p.cmap = _lib.ptr(img), _lib.ptr(cmap)
    p.fromrgb_w, p.fromrgb_b = _lib.ptr(ws[0]), _lib.ptr(ws[1])
    for i in range(nb):
        blk = ws[2 + 5 * i: 7 + 5 * i]
        for name, t in zip(('conv0_w', 'conv0_b', 'conv1_w', 'conv1_b', 'skip_w'), blk):
            getattr(p, name)[i] = t.data_ptr()
    tail = ws[2 + 5 * nb:]
    (p.b4_conv_w, p.b4_conv_b, p.fc_w, p.fc_b, p.out_w, p.out_b) = [_lib.ptr(t) for t in tail]
    return p


def _forward(save, img, cmap, ws):
    """nfi_disc_forward on (img, cmap, ws) -> (state, logits [B,1]); state = (params, workspace,
    the contiguous tensors behind the params' pointers, logits), what the backward passes read."""
    tensors = [t for t in (img, cmap) + tuple(ws) if t is not None]
    if not all(t.is_cuda for t in tensors):
        raise _lib.NfiError('fused discriminator: only runs on CUDA tensors (there is no CPU path)')
    if not all(t.dtype == torch.float32 for t in tensors):
        raise _lib.NfiError('fused discriminator: fp32 images and parameters only, got %s'
                            % sorted({str(t.dtype) for t in tensors}))
    dev = img.device
    if any(t.device != dev for t in tensors):
        raise _lib.NfiError('fused discriminator: image, cmap and parameters on different devices')
    B = img.shape[0]
    lib = _lib.load()
    with torch.cuda.device(dev):
        ic = img.detach().contiguous()
        cc = cmap.detach().contiguous() if cmap is not None else None
        wc = [t.detach().contiguous() for t in ws]
        out = torch.empty(B, 1, device=dev)
        p = _params(ic, cc, wc, save)
        p.logits = _lib.ptr(out)
        nbytes = lib.nfi_disc_workspace_bytes(ctypes.byref(p))
        if nbytes == 0:
            raise _lib.NfiError('fused discriminator: sizes outside the kernels\' envelope (B %d, '
                                'image %s)' % (B, tuple(img.shape)))
        work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        p.workspace, p.workspace_bytes = work.data_ptr(), nbytes
        _lib.check(lib.nfi_disc_forward(ctypes.byref(p), _lib.stream(dev)))
    return (p, work, ic, cc, wc, out), out


class _DiscFunction(torch.autograd.Function):
    """(save, img, cmap or None, backbone weights / biases) -> logits [B,1]."""

    @staticmethod
    def forward(ctx, save, img, cmap, *ws):
        state, out = _forward(save, img, cmap, ws)
        # the backward reads the workspace and the tensors behind p's pointers
        ctx.state = state if save else None
        return out

    @staticmethod
    def backward(ctx, g_logits):
        state = _lib.take_saved(ctx, 'discriminator')
        return (None, *_backward(state, g_logits, ctx.needs_input_grad[1:]))


def _backward(state, g_logits, needs):
    """nfi_disc_backward on a saved forward: the gradients (image, cmap, every weight; None where
    ``needs``, one flag per input, says not) of sum(g_logits * logits)."""
    p, work, ic, cc, wc, out = state
    dev = work.device
    with torch.cuda.device(dev):
        gi, gc, gw, g = _grad_outputs(state, needs)
        gl = g_logits.detach().to(torch.float32).reshape(-1).contiguous()
        _lib.check(_lib.load().nfi_disc_backward(ctypes.byref(p), _lib.ptr(gl), _lib.ptr(gi), _lib.ptr(gc),
                                                 ctypes.byref(g), _lib.stream(dev)))
    return (gi, gc, *gw)


class _R1Link:
    """The saved forward of one R1-shaped call, shared by the three passes that read it: the
    create_graph backward (``graph``), the HVP of its image gradient (``hvp``) and the plain
    backward (``plain``).  The workspace is released once no pass can still come: after a plain
    backward that ran first (the call never took the penalty), or after the plain backward and the
    HVP, in either order."""

    def __init__(self, state, ctx):
        self.state, self.ctx = state, ctx
        self.graph = self.hvp = self.plain = False

    def release(self):
        self.state = None
        if self.ctx is not None:
            self.ctx.state, self.ctx = None, None

    def take(self, what):
        if self.state is None:
            raise _lib.NfiError('fused discriminator (R1): %s after the workspace was released (a plain '
                                'backward that ran first, or both the plain backward and the HVP, '
                                'have run)' % what)
        return self.state


class _DiscR1Function(torch.autograd.Function):
    """(img, cmap or None, backbone weights / biases) -> logits [B,1] of an R1-shaped call.  Its
    backward under create_graph returns the gradients through ``_DiscGradFunction`` (so the image
    gradient can be differentiated again); without, it is the first-order backward."""

    @staticmethod
    def forward(ctx, img, cmap, *ws):
        state, out = _forward(1, img, cmap, ws)
        ctx.link = _R1Link(state, ctx)
        ctx.state = state   # (what saved_preactivations finds)
        ctx.save_for_backward(img, cmap, *ws)
        return out

    @staticmethod
    def backward(ctx, g_logits):
        link = ctx.link
        needs = ctx.needs_input_grad
        if torch.is_grad_enabled():
            if link.graph:
                raise _lib.NfiError('fused discriminator (R1): a second create_graph backward of one '
                                    'forward is not supported')
            link.take('create_graph backward')
            link.graph = True
            img, cmap, *ws = ctx.saved_tensors
            grads = _DiscGradFunction.apply(link, needs, g_logits, img, cmap, *ws)
            return tuple(g if n else None for g, n in zip(grads, needs))
        if link.plain:
            raise _lib.NfiError('fused discriminator (R1): a second plain backward of one forward is not '
                                'supported (retain_graph)')
        state = link.take('plain backward')
        link.plain = True
        grads = _backward(state, g_logits, needs)
        if not link.graph or link.hvp:
            link.release()
        return grads


class _DiscGradFunction(torch.autograd.Function):
    """(link, needs, g_logits, img, cmap, weights) -> the first-order gradients (image, cmap, every
    weight; None where ``needs`` says not) of sum(g_logits * logits): forward ``nfi_disc_backward``, backward ``nfi_disc_backward_hvp`` on
    the image gradient's cotangent.  Only the image gradient may be differentiated again."""

    @staticmethod
    def forward(ctx, link, needs, g_logits, img, cmap, *ws):
        ctx.set_materialize_grads(False)
        ctx.link = link
        ctx.n_ws = len(ws)
        ctx.save_for_backward(g_logits)
        return _backward(link.state, g_logits, needs)

    @staticmethod
    def backward(ctx, t_img, *rest):
        if torch.is_grad_enabled():
            raise _lib.NfiError('fused discriminator (R1): the HVP is not differentiable (a third '
                                'derivative)')
        if any(d is not None and bool(d.any()) for d in rest):
            raise _lib.NfiError('fused discriminator (R1): only the image gradient can be differentiated '
                                'again (a cotangent reached the cmap or parameter gradients)')
        link = ctx.link
        if link.hvp:
            raise _lib.NfiError('fused discriminator (R1): a second HVP of one forward is not supported')
        none = (None,) * (5 + ctx.n_ws)
        if t_img is None:
            return none
        state = link.take('HVP')
        link.hvp = True
        g_logits, = ctx.saved_tensors
        needs = ctx.needs_input_grad
        try:
            grads = _hvp(state, g_logits, t_img, needs[2], needs[3:])
        finally:
            if link.plain:
                link.release()
        return (None, None, *grads)


def _hvp(state, g_logits, t_img, need_gl, needs):
    """nfi_disc_backward_hvp: the gradients (g_logits, image, cmap, every weight) of
    <t_img, d(sum g_logits logits)/dimg>; its scratch lives for the call."""
    p, work, ic, cc, wc, out = state
    dev = work.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        gl = g_logits.detach().to(torch.float32).reshape(-1).contiguous()
        t = t_img.detach().to(torch.float32).contiguous()
        g_gl = torch.zeros_like(gl) if need_gl else None
        gi, gc, gw, g = _grad_outputs(state, needs)
        nbytes = lib.nfi_disc_r1_scratch_bytes(ctypes.byref(p))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        h = _lib.DiscHvp(g_logits=gl.data_ptr(), t_img=t.data_ptr(), scratch=scratch.data_ptr(),
                         scratch_bytes=nbytes, grad_img=_lib.ptr(gi), grad_cmap=_lib.ptr(gc),
                         grad_g_logits=_lib.ptr(g_gl))
        _lib.check(lib.nfi_disc_backward_hvp(ctypes.byref(p), ctypes.byref(h), ctypes.byref(g), _lib.stream(dev)))
        del scratch
    return ((g_gl.view_as(g_logits) if g_gl is not None else None), gi, gc, *gw)


def _grad_outputs(state, needs):
    """The zeroed ``+=`` outputs of a backward pass on ``state``'s forward: image, cmap and every
    weight (None where ``needs``, one flag per input, says not), and the weights' ``DiscGrads``."""
    p, work, ic, cc, wc, out = state
    gi = torch.zeros_like(ic) if needs[0] else None
    gc = torch.zeros_like(cc) if (cc is not None and needs[1]) else None
    gw = [torch.zeros_like(t) if needs[2 + i] else None for i, t in enumerate(wc)]
    return gi, gc, gw, _params_grads(gw, p.resolution)


def _params_grads(gw, R):
    nb = len(block_resolutions(R))
    g = _lib.DiscGrads()
    g.fromrgb_w, g.fromrgb_b = _lib.ptr(gw[0]), _lib.ptr(gw[1])
    for i in range(nb):
        blk = gw[2 + 5 * i: 7 + 5 * i]
        for name, t in zip(('conv0_w', 'conv0_b', 'conv1_w', 'conv1_b', 'skip_w'), blk):
            getattr(g, name)[i] = t.data_ptr() if t is not None else 0
    (g.b4_conv_w, g.b4_conv_b, g.fc_w, g.fc_b, g.out_w, g.out_b) = [_lib.ptr(t) for t in gw[2 + 5 * nb:]]
    return g


def saved_preactivations(out):
    """The pre-activations (or same-signed activations) the saved forward behind ``out`` (logits of
    a call that requires grad, before its backward has run) keeps, fp32: a dict of 'fromrgb'
    [B,R,R,C], ('conv0', r) [B,r,r,C] and ('conv1', r) [B,r/2,r/2,C'] channel-last, 'b4.conv'
    [B,512,4,4] and 'b4.fc' [B,512].  Where a value is positive the backward takes the leaky
    ReLU's unit-slope branch; tests read the branches from them."""
    p, work = _lib.find_saved(out, 'discriminator')[:2]
    dev = work.device
    lib = _lib.load()
    B, R = p.batch, p.resolution
    rs = block_resolutions(R)
    res = {}
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)

        def get(block, which, shape):
            t = torch.empty(shape, device=dev)
            _lib.check(lib.nfi_disc_saved_preactivation(ctypes.byref(p), block, which, _lib.ptr(t), stream))
            return t

        res['fromrgb'] = get(0, 0, (B, R, R, channels(R)))
        for i, r in enumerate(rs):
            res[('conv0', r)] = get(i, 1, (B, r, r, channels(r)))
            res[('conv1', r)] = get(i, 2, (B, r // 2, r // 2, channels(r // 2)))
        res['b4.conv'] = get(len(rs), 0, (B, C4, 4, 4))
        res['b4.fc'] = get(len(rs), 1, (B, C4))
    return res


def _weights(module):
    """The weights and biases the forward reads, by attribute.  ``module.parameters()`` will not do:
    an ``nn.DataParallel`` replica has no registered parameters, its weights are plain tensor
    attributes (``Module._replicate_for_data_parallel``, ``replicate()``)."""
    for m in module.modules():
        for name in ('weight', 'bias'):
            t = getattr(m, name, None)
            if torch.is_tensor(t):
                yield t


def _fused_forward(self, x, iteration, pose=None, image=None, focal=None):
    """Discriminator.forward (discriminator.py:57-80) with the backbone on nfi_disc_forward."""
    unfused = self._nfi_unfused_class.forward
    bb = self.backbone
    grad = torch.is_grad_enabled()
    r1_shaped = grad and x.requires_grad and any(t.requires_grad for t in _weights(self))
    r1 = r1_shaped and getattr(self, '_nfi_r1', False)
    if ((r1_shaped and not r1) or self.use_encoder or self.num_classes or x.dim() != 4 or x.shape[0] % 4 != 0
            or x.shape[1] != bb.img_channels or tuple(x.shape[2:]) != (bb.img_resolution,) * 2
            or not _layout_ok(bb)):
        return unfused(self, x, iteration, pose, image, focal)
    cmap = None
    if self.conditional_pose:
        pose_utils = sys.modules[self._nfi_unfused_class.__module__].pose_utils
        cond = pose_utils.matrix_to_conditioning_vector(pose, focal, self.dataset_config['camera_flipped'])
        cmap = bb.mapping(None, cond)
    elif bb.c_dim > 0:
        return unfused(self, x, iteration, pose, image, focal)
    return logits(bb, x, cmap, r1=r1)


def enable_fused_discriminator(discriminator, enabled=True, r1=False):
    """Switches a reference ``Discriminator`` instance to the fused backbone (``enabled=False``
    switches it back); returns the instance.  ``r1=True`` also runs R1-shaped calls on the kernels,
    their double backward on ``nfi_disc_backward_hvp``; the flag is an instance attribute, so
    ``nn.DataParallel``'s replicas (which copy the instance's ``__dict__``) keep it."""
    m = _lib.switch_class(discriminator, _fused_forward, enabled)
    if enabled and r1:
        m._nfi_r1 = True
    else:
        m.__dict__.pop('_nfi_r1', None)
    return m
