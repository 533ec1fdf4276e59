"""Generator front-end with the plane producer on sm_90a.

``FusedGeneratorFront(G)`` is the part of the reference's ``Generator.forward``
(/root/reference/models/generator.py:407-477,500-502) that turns the model input into the
radiance field -- latent selection / mapping network, palette (texture mapper), synthesis
network -- with the synthesis network run by ``synthesis.FusedSynthesis`` (wgmma kernels,
planes emitted channel-last).  ``G`` stays the reference's own module and the owner of every
parameter; its tiny MLPs (mapping network, texture mapper, encoder) run as they are.

It returns the reference's ``model_outputs`` dict with a ``'triplane'`` entry instead of the
``'sampler'`` closure: ``render.render`` hands that entry to the fused render kernels, which is
what it would have done with the closure's captured planes anyway (render.extract_field).

Envelope: requests within {'sampler', 'attention_values'} under ``torch.no_grad()`` (evaluation
renders, encoder-training targets, visualisation).  The regulariser heads and every call that
differentiates through the synthesis network are the reference module's; ``render`` picks this
front-end only when a call is inside the envelope (``render.enable_fused_synthesis``).

``FusedInversionFront(G)`` is the same front-end for grad-enabled calls with a frozen synthesis
network -- the inversion loop, which differentiates the render to the latents (and the pose):
the planes come from ``FusedSynthesis.forward_differentiable``, whose backward carries dL/dplanes
to ws on the sm_90a kernels.  Mapping network, texture mapper and the ``expand`` of [B,1,512]
latents stay torch autograd.  ``render`` picks it with ``render.enable_fused_inversion``.

``GeneratorStepFront(G)`` is ``HeadsGeneratorFront``'s body (regulariser heads on the fused point
evaluator) for grad-enabled calls with a trainable synthesis network -- the GAN generator step and
the SDF pre-training step -- with the planes from ``FusedSynthesis.forward_trainable``.
``render`` (and ``ParallelModel``'s ``pretrain_sdf`` branch) pick it with
``render.enable_fused_generator_step``.
"""
import torch

from . import _lib
from .synthesis import FusedSynthesis

SUPPORTED_OUTPUTS = ('sampler', 'attention_values')
HEAD_OUTPUTS = ('sdf_eikonal_loss', 'sdf_distance_loss', 'total_variation_loss', 'entropy_loss')


def resolve_ws(g, c):
    """Model input -> ws [B,num_ws,512] (generator.py:423-446): z, w (broadcast from one row or
    complete), (z, image) with the encoder, (z, label) with class embeddings."""
    if g.use_encoder:
        z, image = c
        return g.mapping_network(z, g.emb(image)), z.shape[0]
    label = None
    if g.num_classes:
        if isinstance(c, (list, tuple)):
            c, label = c
            assert len(c.shape) == 2
            label = g.class_embedding(label)
        else:
            assert len(c.shape) == 3
    if len(c.shape) == 3:
        ws = (c.expand(-1, g.mapping_network.backbone.num_ws, -1).contiguous()
              if c.shape[1] == 1 else c)
    else:
        ws = g.mapping_network(c, label)
    return ws, c.shape[0]


def resolve_palette(g, ws, request_model_outputs, model_inputs):
    """(attention_values | None, w_synthesis) -- generator.py:452-468."""
    if g.attention_values <= 0:
        return None, ws
    assert ws.shape[1] == 15
    w_tex, w_synthesis = ws[:, 14], ws[:, :14]
    if 'attention_values' in model_inputs:
        attention_values = model_inputs['attention_values']
    elif 'sampler' in request_model_outputs:
        attention_values = g.texture_mapper(w_tex)
        if 'attention_values_bias' in model_inputs:
            attention_values = attention_values + model_inputs['attention_values_bias']
    else:
        attention_values = None
    return attention_values, w_synthesis


def view_conditioning(g, viewdir):
    """--use_viewdir (generator.py:189-253,468-469): the ViewDirectionMapper trunk evaluated on the
    unit view directions [B,H,W,1,3] by the reference module itself -> the 'triplane' entries
    ``render.extract_view`` reads: per-ray features [B,H,W,32] and the effective weights of the
    mapper's output layer."""
    closure = g.viewdir_mapper(viewdir)
    x = dict(zip(closure.__code__.co_freevars,
                 (c.cell_contents for c in closure.__closure__)))['x']
    out = g.viewdir_mapper.output
    return dict(view_features=x.squeeze(-2), w3=out.weight * out.weight_gain,
                b3=out.bias * out.bias_gain)


def decoder_weights(g):
    """EFFECTIVE decoder weights (EqualizedLinear gains applied, differentiably)."""
    l1, l2 = g.decoder.net[0], g.decoder.net[2]
    return (l1.weight * l1.weight_gain, l1.bias * l1.bias_gain,
            l2.weight * l2.weight_gain, l2.bias * l2.bias_gain)


class FusedGeneratorFront:
    def __init__(self, generator):
        self.g = generator
        self.synthesis = FusedSynthesis(generator.synthesis_network)

    @staticmethod
    def supports(request_model_outputs, model_inputs):
        return (not torch.is_grad_enabled()
                and all(o in SUPPORTED_OUTPUTS for o in request_model_outputs)
                and all(k in ('freeze_noise', 'attention_values', 'attention_values_bias')
                        for k in model_inputs))

    def __call__(self, viewdir, c, request_model_outputs=['sampler'], model_inputs={}):
        if not self.supports(request_model_outputs, model_inputs):
            raise _lib.NfiError('FusedGeneratorFront: outside its envelope (no_grad, outputs '
                                'within %r)' % (SUPPORTED_OUTPUTS,))
        return self._outputs(viewdir, c, request_model_outputs, model_inputs, self.synthesis)

    def _outputs(self, viewdir, c, request_model_outputs, model_inputs, synthesis):
        g = self.g
        ws, batch = resolve_ws(g, c)
        attention_values, w_synthesis = resolve_palette(g, ws, request_model_outputs, model_inputs)
        view = view_conditioning(g, viewdir) if (g.use_viewdir and viewdir is not None) else {}
        # ---- planes (generator.py:471-477), channel-last
        noise_mode = 'const' if model_inputs.get('freeze_noise') else 'random'
        planes_cl = synthesis(w_synthesis, noise_mode=noise_mode)
        assert planes_cl.shape[0] == batch
        w1, b1, w2, b2 = decoder_weights(g)
        out = {}
        if 'attention_values' in request_model_outputs:
            assert g.attention_values > 0
            out['attention_values'] = attention_values
        out['triplane'] = dict(
            planes=planes_cl, planes_layout='channel_last', palette=attention_values,
            w1=w1, b1=b1, w2=w2, b2=b2,
            beta=getattr(g, 'beta', None), alpha=getattr(g, 'alpha', None), **view)
        return out


class FusedInversionFront(FusedGeneratorFront):
    """Grad-enabled calls, synthesis network frozen, requests within SUPPORTED_OUTPUTS."""

    def supports(self, request_model_outputs, model_inputs):
        return (torch.is_grad_enabled()
                and not any(p.requires_grad for p in self.g.synthesis_network.parameters())
                and all(o in SUPPORTED_OUTPUTS for o in request_model_outputs)
                and all(k in ('freeze_noise', 'attention_values', 'attention_values_bias')
                        for k in model_inputs))

    def __call__(self, viewdir, c, request_model_outputs=['sampler'], model_inputs={}):
        if not self.supports(request_model_outputs, model_inputs):
            raise _lib.NfiError('FusedInversionFront: outside its envelope (grad enabled, '
                                'synthesis network frozen, outputs within %r)'
                                % (SUPPORTED_OUTPUTS,))
        return self._outputs(viewdir, c, request_model_outputs, model_inputs,
                             self.synthesis.forward_differentiable)


class HeadsGeneratorFront:
    """``Generator.forward`` with autograd intact and the regulariser heads on the fused point
    evaluator (heads.regulariser_heads): the GAN generator step and the SDF pre-training loop
    (run.py:824-868,1007-1044) request 'sdf_eikonal_loss' / 'sdf_distance_loss' /
    'total_variation_loss' / 'entropy_loss' next to the render.  The synthesis network is the
    reference module here (its autograd carries the gradients to the latents / parameters);
    'path_length' (generator.py:484-499) is autograd through it, unchanged.  Same random draws in
    the same order as the reference: synthesis noise, path-length noise, stratified points,
    total-variation perturbation."""

    layout = 'channel_first'   # of the planes _planes returns

    def __init__(self, generator):
        self.g = generator

    def _planes(self, w_synthesis, batch, model_inputs):
        """The plane producer: the reference module, [B,3,32,R,R] channel-first."""
        block_kwargs = {'noise_mode': 'const'} if model_inputs.get('freeze_noise') else {}
        planes = self.g.synthesis_network(w_synthesis, **block_kwargs)
        return planes.view(batch, 3, 32, planes.shape[-2], planes.shape[-1])

    def _path_length(self, ws, planes, attention_values):
        """generator.py:484-499: autograd through the reference module, create_graph."""
        import math
        g = self.g
        pl_noise = torch.randn_like(planes) / math.sqrt(planes.shape[-2] * planes.shape[-1])
        target = (planes * pl_noise).sum()
        if g.attention_values > 0:
            target = target + (attention_values * torch.randn_like(attention_values)).sum()
        pl_grad, = torch.autograd.grad(target, inputs=ws, create_graph=True)
        return pl_grad.square().sum(dim=-1).mean(dim=-1).sqrt()

    @staticmethod
    def supports(request_model_outputs, model_inputs):
        return (any(o in HEAD_OUTPUTS for o in request_model_outputs)
                and all(o in SUPPORTED_OUTPUTS + HEAD_OUTPUTS + ('path_length',)
                        for o in request_model_outputs))

    def __call__(self, viewdir, c, request_model_outputs=['sampler'], model_inputs={}):
        from .heads import regulariser_heads
        g = self.g
        # (the heads read the distance row of the decoder only: nothing view-dependent, 520-585)
        view = view_conditioning(g, viewdir) if (g.use_viewdir and viewdir is not None) else {}
        ws, batch = resolve_ws(g, c)
        if 'path_length' in request_model_outputs:
            assert torch.is_grad_enabled()
            ws = ws.contiguous().requires_grad_()
        attention_values, w_synthesis = resolve_palette(g, ws, request_model_outputs, model_inputs)
        planes = self._planes(w_synthesis, batch, model_inputs)
        out = {}
        if 'attention_values' in request_model_outputs:
            assert g.attention_values > 0
            out['attention_values'] = attention_values
        if 'path_length' in request_model_outputs:   # generator.py:484-499
            out['path_length'] = self._path_length(ws, planes, attention_values)
        w1, b1, w2, b2 = decoder_weights(g)
        out.update(regulariser_heads(planes, w1, b1, w2, b2, getattr(g, 'beta', None),
                                     g.scene_range, request_model_outputs, use_sdf=g.use_sdf,
                                     training=g.training, layout=self.layout))
        if 'sampler' in request_model_outputs:
            out['triplane'] = dict(planes=planes, planes_layout=self.layout,
                                   palette=attention_values, w1=w1, b1=b1, w2=w2, b2=b2,
                                   beta=getattr(g, 'beta', None), alpha=getattr(g, 'alpha', None),
                                   **view)
        return out


class GeneratorStepFront(HeadsGeneratorFront):
    """The GAN generator step and the SDF pre-training step with the plane producer on sm_90a:
    ``HeadsGeneratorFront``'s body with the planes from ``FusedSynthesis.forward_trainable``
    (channel-last; the heads and the render read that layout), whose backward carries dL/dplanes
    to ws and to every synthesis parameter.  Envelope: grad enabled, a synthesis parameter
    requires grad, requests within SUPPORTED_OUTPUTS + HEAD_OUTPUTS ('path_length' is a double
    backward through the synthesis network: it keeps the reference module).  It does not overlap
    ``FusedGeneratorFront`` (no_grad) or ``FusedInversionFront`` (frozen synthesis).  Same random
    draws in the same order as the reference: synthesis noise, stratified points, total-variation
    perturbation.  ``render`` picks it with ``render.enable_fused_generator_step``."""

    layout = 'channel_last'

    def __init__(self, generator):
        super().__init__(generator)
        self.synthesis = FusedSynthesis(generator.synthesis_network)

    def _planes(self, w_synthesis, batch, model_inputs):
        noise_mode = 'const' if model_inputs.get('freeze_noise') else 'random'
        planes_cl = self.synthesis.forward_trainable(w_synthesis, noise_mode=noise_mode)
        assert planes_cl.shape[0] == batch
        return planes_cl

    def supports(self, request_model_outputs, model_inputs):
        return (torch.is_grad_enabled()
                and any(p.requires_grad for p in self.g.synthesis_network.parameters())
                and all(o in SUPPORTED_OUTPUTS + HEAD_OUTPUTS for o in request_model_outputs)
                and all(k in ('freeze_noise', 'attention_values', 'attention_values_bias')
                        for k in model_inputs))

    def __call__(self, viewdir, c, request_model_outputs=['sampler'], model_inputs={}):
        if not self.supports(request_model_outputs, model_inputs):
            raise _lib.NfiError('GeneratorStepFront: outside its envelope (grad enabled, a '
                                'trainable synthesis network, outputs within %r)'
                                % (SUPPORTED_OUTPUTS + HEAD_OUTPUTS,))
        return super().__call__(viewdir, c, request_model_outputs, model_inputs)


class PathLengthGeneratorStepFront(GeneratorStepFront):
    """``GeneratorStepFront`` for the requests that also ask for 'path_length' -- the first
    generator call of every G-step of the documented training recipe (run.py:970-986 with
    --path_length_regularization).  The planes and the synthesis rows of the path-length gradient
    come from ``FusedSynthesis.forward_trainable_with_path_length`` (its double backward is the
    fused HVP); row 14 (the texture latent, read by the attention palette only) is autograd through
    the texture mapper, create_graph, and ppl is formed as generator.py:498.  Same random draws in
    the same order as the reference: synthesis noise, path-length noise, attention noise,
    stratified points, total-variation perturbation.  ``render`` picks it with
    ``render.enable_fused_path_length``."""

    def _planes(self, w_synthesis, batch, model_inputs):
        noise_mode = 'const' if model_inputs.get('freeze_noise') else 'random'
        planes_cl, self._pl_grad = self.synthesis.forward_trainable_with_path_length(
            w_synthesis, noise_mode=noise_mode)
        assert planes_cl.shape[0] == batch
        return planes_cl

    def _path_length(self, ws, planes, attention_values):
        g = self.g
        pl_grad, self._pl_grad = self._pl_grad, None
        if g.attention_values > 0:   # ws[:, 14] is w_tex; the synthesis reads ws[:, :14]
            target = (attention_values * torch.randn_like(attention_values)).sum()
            g_tex = None
            if target.requires_grad:
                g_tex, = torch.autograd.grad(target, inputs=ws, create_graph=True, allow_unused=True)
            row = g_tex[:, 14:] if g_tex is not None else torch.zeros_like(ws[:, 14:])
            pl_grad = torch.cat([pl_grad, row], dim=1)
        return pl_grad.square().sum(dim=-1).mean(dim=-1).sqrt()

    def supports(self, request_model_outputs, model_inputs):
        return (torch.is_grad_enabled()
                and 'path_length' in request_model_outputs
                and any(p.requires_grad for p in self.g.synthesis_network.parameters())
                and all(o in SUPPORTED_OUTPUTS + HEAD_OUTPUTS + ('path_length',)
                        for o in request_model_outputs)
                and all(k in ('freeze_noise', 'attention_values', 'attention_values_bias')
                        for k in model_inputs))

    def __call__(self, viewdir, c, request_model_outputs=['sampler'], model_inputs={}):
        if not self.supports(request_model_outputs, model_inputs):
            raise _lib.NfiError('PathLengthGeneratorStepFront: outside its envelope (grad '
                                "enabled, a trainable synthesis network, 'path_length' requested, "
                                'outputs within %r)' % (SUPPORTED_OUTPUTS + HEAD_OUTPUTS
                                                        + ('path_length',),))
        return HeadsGeneratorFront.__call__(self, viewdir, c, request_model_outputs, model_inputs)
