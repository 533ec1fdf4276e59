"""Drop-in for the reference's per-ray render: same call, fused CUDA underneath.

``render`` has the signature, argument meaning, return tuple and error
behaviour of /root/reference/run.py:176-350, and ``ParallelModel`` mirrors
run.py:560-617, so the GAN-training and inversion loops of run.py call them
unchanged (INTEGRATION.md shows the two-line patch).  Like the reference
function, ``render`` reads two module globals that the host script sets:

    args            .use_viewdir .use_sdf .attention_values .fine_sampling
    dataset_config  ['scene_range'] ['white_background']

(``configure(args, dataset_config)`` sets both).  ``target_model`` is the
reference's own ``models.generator.Generator`` (unmodified): it still runs
the mapping / texture-mapper / synthesis front-end and hands back its
``sampler`` closure; instead of CALLING that closure (which would materialise
the [B, H*W*S, .] tensors of models/generator.py:587-681) the tri-planes,
palette and decoder weights it closes over are passed to the fused kernels.

Randomness: the reference draws ``torch.rand_like(depth_values)`` before the
generator forward and ``torch.rand([rays, S])`` after it
(lib/nerf_utils.py:112,201).  ``render`` makes the same two draws, in the same
order and shapes, from the same default CUDA generator, so a seeded run
consumes the generator exactly like the reference does.
"""

import types

import torch
from torch import nn

from . import _lib
from .fused import RenderConfig, fused_render
from .rays import unit_rays

args = None
dataset_config = None
depth_samples_per_ray = 64  # run.py:511


def configure(new_args, new_dataset_config, samples_per_ray=None):
    """Sets the module globals ``render`` reads (run.py does this by being a
    script; here the host calls it once after parsing its arguments)."""
    global args, dataset_config, depth_samples_per_ray
    if isinstance(new_args, dict):
        new_args = types.SimpleNamespace(**new_args)
    for k in ('use_viewdir', 'use_sdf', 'attention_values', 'fine_sampling'):
        if not hasattr(new_args, k):
            raise AttributeError('args.%s is required (run.py:216-259)' % k)
    for k in ('scene_range', 'white_background'):
        if k not in new_dataset_config:
            raise KeyError('dataset_config[%r] is required (run.py:200,348)' % k)
    args = new_args
    dataset_config = new_dataset_config
    if samples_per_ray is not None:
        depth_samples_per_ray = samples_per_ray


_FRONTS = {}
_INV_FRONTS = {}
_HEAD_FRONTS = {}
_GEN_FRONTS = {}
_PL_FRONTS = {}


def enable_fused_heads(target_model, enabled=True):
    """Makes ``render`` (and ``ParallelModel``'s SDF pre-training branch) compute the regulariser
    outputs of ``target_model`` -- 'sdf_eikonal_loss', 'sdf_distance_loss',
    'total_variation_loss', 'entropy_loss' (generator.py:520-585) -- with the fused point
    evaluator instead of the unfused decoder + double backward."""
    from .generator import HeadsGeneratorFront
    if enabled:
        _HEAD_FRONTS[id(target_model)] = HeadsGeneratorFront(target_model)
    else:
        _HEAD_FRONTS.pop(id(target_model), None)


def enable_fused_synthesis(target_model, enabled=True):
    """Makes ``render`` produce ``target_model``'s tri-planes with the sm_90a synthesis
    kernels (generator.FusedGeneratorFront) for the calls inside their envelope: under
    ``torch.no_grad()`` and without regulariser outputs.  Every other call keeps running the
    reference module's own forward (it needs autograd through the synthesis network)."""
    from .generator import FusedGeneratorFront
    if enabled:
        _FRONTS[id(target_model)] = FusedGeneratorFront(target_model)
    else:
        _FRONTS.pop(id(target_model), None)


def enable_fused_inversion(target_model, enabled=True):
    """Makes ``render`` produce ``target_model``'s tri-planes with the sm_90a synthesis kernels
    for grad-enabled calls too, when the synthesis network is frozen (the inversion loop:
    gradients to the latents and the pose, generator.FusedInversionFront); the planes' gradient
    goes back to ws through the fused synthesis backward.  A call with a trainable synthesis
    parameter, or with regulariser outputs, keeps running the reference module.  Calls under
    ``torch.no_grad()`` are ``enable_fused_synthesis``'s."""
    from .generator import FusedInversionFront
    if enabled:
        _INV_FRONTS[id(target_model)] = FusedInversionFront(target_model)
    else:
        _INV_FRONTS.pop(id(target_model), None)


def enable_fused_generator_step(target_model, enabled=True):
    """Makes ``render`` (and ``ParallelModel``'s SDF pre-training branch) produce
    ``target_model``'s tri-planes with the sm_90a synthesis kernels, forward and backward to ws and
    to every synthesis parameter, for grad-enabled calls with a trainable synthesis network and
    requests within SUPPORTED_OUTPUTS + HEAD_OUTPUTS (generator.GeneratorStepFront: the GAN
    generator step, the dual discriminator's second call, SDF pre-training).  'path_length' and
    calls outside that envelope route as before."""
    from .generator import GeneratorStepFront
    if enabled:
        _GEN_FRONTS[id(target_model)] = GeneratorStepFront(target_model)
    else:
        _GEN_FRONTS.pop(id(target_model), None)


def enable_fused_path_length(target_model, enabled=True):
    """Makes ``render`` run ``target_model``'s generator calls that request 'path_length' (the
    path-length regulariser, generator.py:484-499: the first G call of every generator step
    with --path_length_regularization) on the sm_90a synthesis kernels, the regulariser's double
    backward included (generator.PathLengthGeneratorStepFront).  It applies to grad-enabled calls
    with a trainable synthesis network and requests within SUPPORTED_OUTPUTS + HEAD_OUTPUTS +
    'path_length'; every other call routes as without it."""
    from .generator import PathLengthGeneratorStepFront
    if enabled:
        _PL_FRONTS[id(target_model)] = PathLengthGeneratorStepFront(target_model)
    else:
        _PL_FRONTS.pop(id(target_model), None)


def _closure_vars(fn):
    out = {}
    for name, cell in zip(fn.__code__.co_freevars, fn.__closure__ or ()):
        try:
            out[name] = cell.cell_contents
        except ValueError:  # never assigned (e.g. attention_values when A == 0)
            out[name] = None
    return out


def _join_planes(xy, xz, yz):
    """[B,32,R,R] x3 -> [B,3,32,R,R] without a copy when the three are the
    slices ``planes[:, i]`` of one synthesis output (generator.py:475-502)."""
    B, C, R, _ = xy.shape
    base = xy._base
    if (base is not None and xz._base is base and yz._base is base
            and base.is_contiguous() and base.numel() == 3 * xy.numel()
            and xy.stride() == xz.stride() == yz.stride() == (3 * C * R * R, R * R, R, 1)
            and xy.data_ptr() == base.data_ptr()
            and xz.data_ptr() == base.data_ptr() + 4 * C * R * R
            and yz.data_ptr() == base.data_ptr() + 8 * C * R * R):
        return base.view(B, 3, C, R, R)
    return torch.stack((xy, xz, yz), dim=1)


def extract_view(target_model, sampler):
    """--use_viewdir (generator.py:189-253,468-469,662-663): the per-ray features ``x``
    [B,H,W,1,32] the ViewDirectionMapper trunk produced from the view directions (captured by
    the mapper closure the sampler closes over) and the effective weights of its output layer.
    Returns (view_features [B,H,W,32], w3, b3)."""
    if isinstance(sampler, dict):
        return sampler['view_features'], sampler['w3'], sampler['b3']
    mapper_closure = _closure_vars(sampler).get('viewdir_mapper_closure')
    if mapper_closure is None:
        raise _lib.NfiError("args.use_viewdir is set but target_model's sampler carries no "
                            'viewdir_mapper_closure (generator.py:468-469): was the model built '
                            'with use_viewdir=True?')
    x = _closure_vars(mapper_closure)['x']
    out = target_model.viewdir_mapper.output
    return x.squeeze(-2), out.weight * out.weight_gain, out.bias * out.bias_gain


def extract_field(target_model, sampler):
    """Pulls (planes, palette, w1, b1, w2, b2, beta, alpha) out of the
    reference Generator and the sampler closure it returned.

    A model may instead return a dict under ``model_outputs['triplane']`` with
    those keys (no closure introspection needed); ``sampler`` is then that dict.
    """
    if isinstance(sampler, dict):
        f = sampler
        return (f['planes'], f.get('palette'), f['w1'], f['b1'], f['w2'],
                f['b2'], f.get('beta'), f.get('alpha'))  # layout: f.get('planes_layout')
    cv = _closure_vars(sampler)
    for k in ('xy', 'xz', 'yz'):
        if cv.get(k) is None:
            raise _lib.NfiError(
                "target_model's sampler does not close over %r: the fused "
                'renderer needs a reference-style Generator '
                '(models/generator.py:500-502,587)' % k)
    planes = _join_planes(cv['xy'], cv['xz'], cv['yz'])
    palette = cv.get('attention_values')
    dec = target_model.decoder.net
    l1, l2 = dec[0], dec[2]
    # EqualizedLinear: weight * weight_gain, bias * bias_gain (stylegan.py:175-176)
    w1 = l1.weight * l1.weight_gain
    b1 = l1.bias * l1.bias_gain
    w2 = l2.weight * l2.weight_gain
    b2 = l2.bias * l2.bias_gain
    beta = getattr(target_model, 'beta', None)
    alpha = getattr(target_model, 'alpha', None)
    return planes, palette, w1, b1, w2, b2, beta, alpha


def render(target_model,
           height,
           width,
           tform_cam2world,
           focal_length,
           center,
           bbox,
           model_input,
           depth_samples_per_ray,
           randomize=True,
           compute_normals=False,
           compute_semantics=False,
           compute_coords=False,
           extra_model_outputs=[],
           extra_model_inputs={},
           force_no_cam_grad=False):
    """run.py:176-350.  Returns (rgb [B,H,W,3], depth [B,H,W], mask [B,H,W],
    normals|None, semantics-or-coords|None, model_outputs: dict)."""
    if args is None or dataset_config is None:
        raise RuntimeError('call nerf_from_image_b200.render.configure(args, '
                           'dataset_config) first')
    if 'bbox' in extra_model_outputs and compute_coords:
        # models/generator.py:640-657: the closure adds a 100 x box-frame debug density to
        # sigma when coords are requested together with 'bbox'; the fused kernels render
        # without it (the sampler seam, sampler.FusedSampler(bbox_debug=True), has it)
        raise NotImplementedError(
            "'bbox' in extra_model_outputs with compute_coords (the debug box-frame density, "
            'generator.py:640-657) is only available through the sampler seam')
    if compute_normals:
        assert args.use_sdf  # run.py:229
    if compute_semantics:
        assert args.attention_values > 0  # run.py:232
    S = int(depth_samples_per_ray)
    B = tform_cam2world.shape[0]
    dev = tform_cam2world.device
    fine = bool(args.fine_sampling)

    noise_t = noise_u = None
    if randomize:
        noise_t = torch.rand(B, height, width, S, device=dev)

    viewdirs = None
    if args.use_viewdir:
        # run.py:196,210-217: the model is conditioned on the unit ray directions (detached under
        # force_no_cam_grad); its ViewDirectionMapper trunk runs once per ray in the model's own
        # forward, the per-sample part (mapper closure) inside the fused kernels
        _, dirs = unit_rays(height, width, tform_cam2world, focal_length, center, bbox)
        viewdirs = (dirs.detach() if force_no_cam_grad else dirs).unsqueeze(-2)

    requests = ['sampler'] + list(extra_model_outputs)
    front = _FRONTS.get(id(target_model))
    ifront = _INV_FRONTS.get(id(target_model))
    gfront = _GEN_FRONTS.get(id(target_model))
    hfront = _HEAD_FRONTS.get(id(target_model))
    pfront = _PL_FRONTS.get(id(target_model)) if 'path_length' in requests else None
    if pfront is not None and pfront.supports(requests, extra_model_inputs):
        # ... with the path-length regulariser's double backward (PathLengthGeneratorStepFront)
        model_outputs = pfront(viewdirs, model_input, requests, extra_model_inputs)
    elif front is not None and front.supports(requests, extra_model_inputs):
        # plane producer on sm_90a too (generator.FusedGeneratorFront; no_grad calls only)
        model_outputs = front(viewdirs, model_input, requests, extra_model_inputs)
    elif ifront is not None and ifront.supports(requests, extra_model_inputs):
        # ... and its backward to the latents (generator.FusedInversionFront; frozen synthesis)
        model_outputs = ifront(viewdirs, model_input, requests, extra_model_inputs)
    elif gfront is not None and gfront.supports(requests, extra_model_inputs):
        # ... and to the synthesis parameters (generator.GeneratorStepFront; generator step)
        model_outputs = gfront(viewdirs, model_input, requests, extra_model_inputs)
    elif hfront is not None and hfront.supports(requests, extra_model_inputs):
        # regulariser heads on the fused point evaluator (generator.HeadsGeneratorFront)
        model_outputs = hfront(viewdirs, model_input, requests, extra_model_inputs)
    else:
        model_outputs = target_model(viewdirs, model_input, requests, extra_model_inputs)
    sampler = model_outputs.pop('triplane', None) or model_outputs['sampler']
    model_outputs.pop('sampler', None)
    planes, palette, w1, b1, w2, b2, beta, alpha = extract_field(target_model, sampler)
    view = extract_view(target_model, sampler) if args.use_viewdir else None
    layout = sampler.get('planes_layout', 'channel_first') if isinstance(sampler, dict) \
        else 'channel_first'

    if randomize and fine:
        noise_u = torch.rand(B * height * width, S, device=dev)

    cfg = RenderConfig(scene_range=float(dataset_config['scene_range']),
                       white_background=bool(dataset_config['white_background']),
                       use_sdf=bool(args.use_sdf), fine_sampling=fine,
                       attention_values=int(args.attention_values),
                       mlp_mode=int(getattr(args, 'mlp_mode', _lib.MLP_AUTO)))
    extra_mode = _lib.EXTRA_NONE
    if compute_coords:  # coords overwrite semantics, run.py:337-338
        extra_mode = _lib.EXTRA_COORDS
    elif compute_semantics:
        extra_mode = _lib.EXTRA_SEMANTICS

    out = fused_render(
        planes, w1, b1, w2, b2, palette, beta, alpha, tform_cam2world,
        focal_length, center, bbox, cfg, height, width, S, noise_t, noise_u,
        extra_mode, cam_grad=not force_no_cam_grad,
        compute_normals=bool(compute_normals), planes_layout=layout, view=view)
    rgb, depth, mask, extra = out[:4]
    normals = out[4] if compute_normals else None
    return rgb, depth, mask, normals, extra, model_outputs


class ParallelModel(nn.Module):
    """run.py:560-617 with ``render`` above in place of the reference's."""

    def __init__(self, resolution, model=None, model_ema=None, lpips_net=None):
        super().__init__()
        self.resolution = resolution
        self.model = model
        self.model_ema = model_ema
        self.lpips_net = lpips_net

    def forward(self,
                tform_cam2world,
                focal,
                center,
                bbox,
                c,
                use_ema=False,
                ray_multiplier=1,
                res_multiplier=1,
                pretrain_sdf=False,
                compute_normals=False,
                compute_semantics=False,
                compute_coords=False,
                encoder_output=False,
                closure=None,
                closure_params=None,
                extra_model_outputs=[],
                extra_model_inputs={},
                force_no_cam_grad=False):
        model_to_use = self.model_ema if use_ema else self.model
        if pretrain_sdf:
            req = ['sdf_distance_loss', 'sdf_eikonal_loss']
            gfront = _GEN_FRONTS.get(id(model_to_use))
            if gfront is not None and gfront.supports(req, {}):
                return gfront(None, c, request_model_outputs=req)
            hfront = _HEAD_FRONTS.get(id(model_to_use))
            if hfront is not None:
                return hfront(None, c, request_model_outputs=req)
            return model_to_use(None, c, request_model_outputs=req)
        if encoder_output:
            return model_to_use.emb(c)
        res = int(self.resolution * res_multiplier)
        output = render(model_to_use, res, res, tform_cam2world, focal, center,
                        bbox, c, depth_samples_per_ray * ray_multiplier,
                        compute_normals=compute_normals,
                        compute_semantics=compute_semantics,
                        compute_coords=compute_coords,
                        extra_model_outputs=extra_model_outputs,
                        extra_model_inputs=extra_model_inputs,
                        force_no_cam_grad=force_no_cam_grad)
        if closure is not None:
            return closure(self, output[0], output[2], output[4], output[-1],
                           **closure_params)
        return output
