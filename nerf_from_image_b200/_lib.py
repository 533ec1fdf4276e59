"""ctypes binding of libnfi_render.so (the C ABI declared in include/nfi_render.h and the headers
next to it).

The library is built in-tree by ``nerf_from_image_b200/csrc/build.sh`` (or
``__graft_entry__.build()``).  There is no fallback: if the shared object is
missing or a launch fails, the caller gets an exception.
"""

import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# NFI_LIB_PATH points the binding at another build of the same library (A/B timing of two
# builds in one process launch each; tools/time_backward.py) -- never at a different backend.
LIB_PATH = os.environ.get('NFI_LIB_PATH') or os.path.join(_HERE, 'csrc', 'libnfi_render.so')

c_float_p = ctypes.POINTER(ctypes.c_float)
ABI_VERSION = 6  # NFI_ABI_VERSION of include/nfi_render.h
MAX_PEERS = 7
BACKWARD_IMAGES_BYTES = 65536  # the two weight images of a frozen-decoder backward (nfi_layout.h)
BACKWARD_WORKSPACE_BYTES = 65536 + 160 * 32768  # NFI_BACKWARD_WORKSPACE_BYTES
VIEW_BACKWARD_WORKSPACE_BYTES = 98304  # NFI_VIEW_BACKWARD_WORKSPACE_BYTES

EXTRA_NONE, EXTRA_COORDS, EXTRA_SEMANTICS = 0, 1, 2
NOISE_DETERMINISTIC, NOISE_EXPLICIT, NOISE_PHILOX = 0, 1, 2
MLP_AUTO, MLP_FP32_SIMT, MLP_TC_3XTF32, MLP_TC_WARPSPEC, MLP_TC_PIPE = 0, 1, 2, 3, 4


class RenderParams(ctypes.Structure):
    """struct nfi_render_params -- field order must match the header."""
    _fields_ = [
        ('batch', ctypes.c_int32), ('height', ctypes.c_int32),
        ('width', ctypes.c_int32), ('num_samples', ctypes.c_int32),
        ('plane_res', ctypes.c_int32), ('n_attention', ctypes.c_int32),
        ('scene_range', ctypes.c_float),
        ('white_background', ctypes.c_int32), ('use_sdf', ctypes.c_int32),
        ('fine_sampling', ctypes.c_int32), ('noise_mode', ctypes.c_int32),
        ('extra_mode', ctypes.c_int32), ('compute_normals', ctypes.c_int32),
        ('mlp_mode', ctypes.c_int32),
        ('planes', ctypes.c_void_p), ('w1', ctypes.c_void_p),
        ('b1', ctypes.c_void_p), ('w2', ctypes.c_void_p),
        ('b2', ctypes.c_void_p), ('palette', ctypes.c_void_p),
        ('beta', ctypes.c_void_p), ('alpha', ctypes.c_void_p),
        ('c2w', ctypes.c_void_p), ('focal', ctypes.c_void_p),
        ('center', ctypes.c_void_p), ('bbox', ctypes.c_void_p),
        ('noise_t', ctypes.c_void_p), ('noise_u', ctypes.c_void_p),
        ('rgb', ctypes.c_void_p), ('depth', ctypes.c_void_p),
        ('mask', ctypes.c_void_p), ('extra', ctypes.c_void_p),
        ('normals', ctypes.c_void_p), ('z_fine', ctypes.c_void_p),
        ('workspace', ctypes.c_void_p), ('workspace_bytes', ctypes.c_size_t),
        ('noise_seed', ctypes.c_uint64),
        ('n_peers', ctypes.c_int32), ('peer_reserved', ctypes.c_int32),
        ('peer_rgb', ctypes.c_void_p * 7), ('peer_depth', ctypes.c_void_p * 7),
        ('peer_mask', ctypes.c_void_p * 7),
        ('peer_signal', ctypes.c_void_p * 7), ('peer_signal_self', ctypes.c_void_p),
        ('peer_rank', ctypes.c_int32 * 7), ('peer_epoch', ctypes.c_uint32),
        ('peer_done', ctypes.c_void_p),
        ('view_features', ctypes.c_void_p), ('w3', ctypes.c_void_p), ('b3', ctypes.c_void_p),
        ('row_offset', ctypes.c_int32), ('full_height', ctypes.c_int32),
    ]


class RenderGrads(ctypes.Structure):
    """struct nfi_render_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        'g_rgb', 'g_mask', 'g_extra', 'out_rgb', 'out_mask', 'out_extra',
        'grad_planes', 'grad_w1', 'grad_b1', 'grad_w2', 'grad_b2',
        'grad_palette', 'grad_beta', 'grad_alpha', 'grad_origins',
        'grad_dirs', 'grad_view_features', 'grad_w3', 'grad_b3')]


class SampleParams(ctypes.Structure):
    """struct nfi_sample_params."""
    _fields_ = [
        ('batch', ctypes.c_int32), ('plane_res', ctypes.c_int32),
        ('n_attention', ctypes.c_int32), ('use_sdf', ctypes.c_int32),
        ('bbox_debug', ctypes.c_int32), ('scene_range', ctypes.c_float),
        ('n_points', ctypes.c_int64),
    ] + [(n, ctypes.c_void_p) for n in (
        'planes', 'w1', 'b1', 'w2', 'b2', 'palette', 'beta', 'alpha', 'points',
        'sdf_distance', 'sigma', 'rgb', 'semantics', 'normals')]


SYNTH_MAX_BLOCKS = 9


class SynthLayer(ctypes.Structure):
    """struct nfi_synth_layer (include/nfi_synth.h)."""
    _fields_ = [(n, ctypes.c_void_p) for n in ('weight', 'affine_w', 'affine_b', 'bias', 'noise')]


class SynthParams(ctypes.Structure):
    """struct nfi_synth_params."""
    _fields_ = [
        ('batch', ctypes.c_int32), ('img_resolution', ctypes.c_int32),
        ('img_channels', ctypes.c_int32), ('w_dim', ctypes.c_int32),
        ('num_blocks', ctypes.c_int32), ('num_ws', ctypes.c_int32),
        ('channels', ctypes.c_int32 * SYNTH_MAX_BLOCKS),
        ('ws', ctypes.c_void_p), ('const_input', ctypes.c_void_p),
        ('conv0', SynthLayer * SYNTH_MAX_BLOCKS), ('conv1', SynthLayer * SYNTH_MAX_BLOCKS),
        ('torgb', SynthLayer * SYNTH_MAX_BLOCKS),
        ('planes', ctypes.c_void_p), ('workspace', ctypes.c_void_p),
        ('workspace_bytes', ctypes.c_size_t),
    ]


class SynthGrads(ctypes.Structure):
    """struct nfi_synth_grads."""
    _fields_ = [('g_planes', ctypes.c_void_p), ('g_ws', ctypes.c_void_p)]


class SynthLayerGrads(ctypes.Structure):
    """struct nfi_synth_layer_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in ('g_weight', 'g_affine_w', 'g_affine_b', 'g_bias',
                                               'g_noise')]


class SynthParamGrads(ctypes.Structure):
    """struct nfi_synth_param_grads."""
    _fields_ = [
        ('conv0', SynthLayerGrads * SYNTH_MAX_BLOCKS), ('conv1', SynthLayerGrads * SYNTH_MAX_BLOCKS),
        ('torgb', SynthLayerGrads * SYNTH_MAX_BLOCKS), ('g_const', ctypes.c_void_p),
    ]


class SynthHvp(ctypes.Structure):
    """struct nfi_synth_hvp."""
    _fields_ = [('g_planes', ctypes.c_void_p), ('t_ws', ctypes.c_void_p), ('g_ws', ctypes.c_void_p),
                ('scratch', ctypes.c_void_p), ('scratch_bytes', ctypes.c_size_t)]


class SdfPointsParams(ctypes.Structure):
    """struct nfi_sdf_points_params (include/nfi_heads.h)."""
    _fields_ = [('batch', ctypes.c_int32), ('plane_res', ctypes.c_int32),
                ('scene_range', ctypes.c_float), ('n_points', ctypes.c_int64)] + [
        (n, ctypes.c_void_p) for n in ('planes', 'w1', 'b1', 'w2', 'b2', 'points', 'd', 'grad')]


class SdfPointsGrads(ctypes.Structure):
    """struct nfi_sdf_points_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        'g_d', 'g_grad', 'grad_planes', 'grad_w1', 'grad_b1', 'grad_w2_row0', 'grad_b2_0')]


LPIPS_CONVS, LPIPS_TAPS = 13, 5


class LpipsParams(ctypes.Structure):
    """struct nfi_lpips_params (include/nfi_lpips.h)."""
    _fields_ = [
        ('n', ctypes.c_int32), ('height', ctypes.c_int32), ('width', ctypes.c_int32),
        ('save', ctypes.c_int32), ('in0', ctypes.c_void_p), ('in1', ctypes.c_void_p),
        ('conv_w', ctypes.c_void_p * LPIPS_CONVS), ('conv_b', ctypes.c_void_p * LPIPS_CONVS),
        ('lin_w', ctypes.c_void_p * LPIPS_TAPS), ('shift', ctypes.c_void_p),
        ('scale', ctypes.c_void_p), ('out', ctypes.c_void_p), ('workspace', ctypes.c_void_p),
        ('workspace_bytes', ctypes.c_size_t),
    ]


ENCODER_MAPS = 4


class EncoderParams(ctypes.Structure):
    """struct nfi_encoder_params (include/nfi_encoder.h)."""
    _fields_ = [
        ('batch', ctypes.c_int32), ('height', ctypes.c_int32), ('width', ctypes.c_int32),
        ('channels', ctypes.c_int32), ('pose_regressor', ctypes.c_int32),
        ('latent_regressor', ctypes.c_int32), ('save', ctypes.c_int32),
    ] + [(n, ctypes.c_void_p) for n in (
        'features', 'features_latent', 'post0_w', 'post0_b', 'post2_w', 'post2_b', 'post4_w',
        'post4_b', 'wpre_w', 'wpre_b', 'maps', 'pooled', 'workspace')] + [
        ('workspace_bytes', ctypes.c_size_t)]


class EncoderGrads(ctypes.Structure):
    """struct nfi_encoder_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        'g_features', 'g_features_latent', 'g_post0_w', 'g_post0_b', 'g_post2_w', 'g_post2_b',
        'g_post4_w', 'g_post4_b', 'g_wpre_w', 'g_wpre_b')]


DISC_MAX_BLOCKS = 6


class DiscParams(ctypes.Structure):
    """struct nfi_disc_params (include/nfi_disc.h)."""
    _fields_ = [(n, ctypes.c_int32) for n in (
        'batch', 'resolution', 'img_channels', 'cmap_dim', 'save')] + [
        (n, ctypes.c_void_p) for n in ('img', 'cmap', 'fromrgb_w', 'fromrgb_b')] + [
        (n, ctypes.c_void_p * DISC_MAX_BLOCKS) for n in (
            'conv0_w', 'conv0_b', 'conv1_w', 'conv1_b', 'skip_w')] + [
        (n, ctypes.c_void_p) for n in (
            'b4_conv_w', 'b4_conv_b', 'fc_w', 'fc_b', 'out_w', 'out_b', 'logits', 'workspace')] + [
        ('workspace_bytes', ctypes.c_size_t)]


class DiscGrads(ctypes.Structure):
    """struct nfi_disc_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in ('fromrgb_w', 'fromrgb_b')] + [
        (n, ctypes.c_void_p * DISC_MAX_BLOCKS) for n in (
            'conv0_w', 'conv0_b', 'conv1_w', 'conv1_b', 'skip_w')] + [
        (n, ctypes.c_void_p) for n in ('b4_conv_w', 'b4_conv_b', 'fc_w', 'fc_b', 'out_w', 'out_b')]


class DiscHvp(ctypes.Structure):
    """struct nfi_disc_hvp (include/nfi_disc_r1.h)."""
    _fields_ = [(n, ctypes.c_void_p) for n in ('g_logits', 't_img', 'scratch')] + [
        ('scratch_bytes', ctypes.c_size_t)] + [
        (n, ctypes.c_void_p) for n in ('grad_img', 'grad_cmap', 'grad_g_logits')]


# every symbol include/nfi_render.h, nfi_synth.h and nfi_heads.h declare (tests/test_abi.py checks
# those headers against this table and the table against the built library); LPIPS_EXPORTS and
# ENCODER_EXPORTS below hold the symbols of include/nfi_lpips.h (tests/test_lpips_abi.py) and
# include/nfi_encoder.h (tests/test_encoder_abi.py), DISC_EXPORTS those of include/nfi_disc.h
# (tests/test_disc_abi.py)
EXPORTS = {
    'nfi_abi_version': (ctypes.c_int, []),
    'nfi_build_info': (ctypes.c_char_p, []),
    'nfi_last_error': (ctypes.c_char_p, []),
    'nfi_render_workspace_bytes': (ctypes.c_size_t,
                                   [ctypes.POINTER(RenderParams)]),
    'nfi_planes_to_channel_last': (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    'nfi_planes_from_channel_last': (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
        ctypes.c_void_p]),
    'nfi_render_forward': (ctypes.c_int, [ctypes.POINTER(RenderParams),
                                          ctypes.c_void_p]),
    'nfi_decoder_forward': (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    'nfi_render_backward': (ctypes.c_int, [ctypes.POINTER(RenderParams),
                                           ctypes.POINTER(RenderGrads),
                                           ctypes.c_void_p]),
    'nfi_render_forward_host': (ctypes.c_int, [ctypes.POINTER(RenderParams),
                                               ctypes.c_int32]),
    'nfi_fill_uniform': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint64,
                                        ctypes.c_uint32, ctypes.c_int64, ctypes.c_void_p]),
    'nfi_sample_field': (ctypes.c_int, [ctypes.POINTER(SampleParams), ctypes.c_void_p]),
    'nfi_sdf_points_forward': (ctypes.c_int, [ctypes.POINTER(SdfPointsParams), ctypes.c_void_p]),
    'nfi_sdf_points_backward': (ctypes.c_int, [ctypes.POINTER(SdfPointsParams),
                                               ctypes.POINTER(SdfPointsGrads), ctypes.c_void_p]),
    'nfi_synthesis_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(SynthParams)]),
    'nfi_synthesis_forward': (ctypes.c_int, [ctypes.POINTER(SynthParams), ctypes.c_void_p]),
    'nfi_synthesis_saved_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(SynthParams)]),
    'nfi_synthesis_forward_saved': (ctypes.c_int, [ctypes.POINTER(SynthParams), ctypes.c_void_p]),
    'nfi_synthesis_backward': (ctypes.c_int, [ctypes.POINTER(SynthParams),
                                              ctypes.POINTER(SynthGrads), ctypes.c_void_p]),
    'nfi_synthesis_saved_preactivation': (ctypes.c_int, [ctypes.POINTER(SynthParams),
                                                         ctypes.c_int32, ctypes.c_int32,
                                                         ctypes.c_void_p, ctypes.c_void_p]),
    'nfi_synthesis_param_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(SynthParams)]),
    'nfi_synthesis_backward_params': (ctypes.c_int, [ctypes.POINTER(SynthParams),
                                                     ctypes.POINTER(SynthGrads),
                                                     ctypes.POINTER(SynthParamGrads),
                                                     ctypes.c_void_p]),
    'nfi_synthesis_hvp_scratch_bytes': (ctypes.c_size_t, [ctypes.POINTER(SynthParams)]),
    'nfi_synthesis_backward_hvp': (ctypes.c_int, [ctypes.POINTER(SynthParams),
                                                  ctypes.POINTER(SynthHvp),
                                                  ctypes.POINTER(SynthParamGrads),
                                                  ctypes.c_void_p]),
    'nfi_pose_to_matrix': (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'nfi_pose_to_matrix_backward': (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
}

LPIPS_EXPORTS = {
    'nfi_lpips_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(LpipsParams)]),
    'nfi_lpips_forward': (ctypes.c_int, [ctypes.POINTER(LpipsParams), ctypes.c_void_p]),
    'nfi_lpips_backward': (ctypes.c_int, [ctypes.POINTER(LpipsParams), ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'nfi_lpips_saved_preactivation': (ctypes.c_int, [ctypes.POINTER(LpipsParams), ctypes.c_int32,
                                                     ctypes.c_void_p, ctypes.c_void_p]),
}

ENCODER_EXPORTS = {
    'nfi_encoder_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(EncoderParams)]),
    'nfi_encoder_forward': (ctypes.c_int, [ctypes.POINTER(EncoderParams), ctypes.c_void_p]),
    'nfi_encoder_backward': (ctypes.c_int, [ctypes.POINTER(EncoderParams), ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.POINTER(EncoderGrads),
                                            ctypes.c_void_p]),
    'nfi_encoder_saved_activation': (ctypes.c_int, [ctypes.POINTER(EncoderParams), ctypes.c_int32,
                                                    ctypes.c_void_p, ctypes.c_void_p]),
}

DISC_EXPORTS = {
    'nfi_disc_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(DiscParams)]),
    'nfi_disc_forward': (ctypes.c_int, [ctypes.POINTER(DiscParams), ctypes.c_void_p]),
    'nfi_disc_backward': (ctypes.c_int, [ctypes.POINTER(DiscParams), ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.POINTER(DiscGrads), ctypes.c_void_p]),
    'nfi_disc_saved_preactivation': (ctypes.c_int, [ctypes.POINTER(DiscParams), ctypes.c_int32,
                                                    ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
}

# include/nfi_disc_r1.h (tests/test_disc_r1_abi.py)
DISC_R1_EXPORTS = {
    'nfi_disc_r1_scratch_bytes': (ctypes.c_size_t, [ctypes.POINTER(DiscParams)]),
    'nfi_disc_backward_hvp': (ctypes.c_int, [ctypes.POINTER(DiscParams), ctypes.POINTER(DiscHvp),
                                             ctypes.POINTER(DiscGrads), ctypes.c_void_p]),
}

SEGFORMER_STAGES, SEGFORMER_MAX_DEPTH, SEGFORMER_DECODER = 4, 64, 768


class SegformerParams(ctypes.Structure):
    """struct nfi_segformer_params (include/nfi_segformer.h)."""
    _fields_ = [('batch', ctypes.c_int32), ('height', ctypes.c_int32), ('width', ctypes.c_int32),
                ('depths', ctypes.c_int32 * SEGFORMER_STAGES), ('out_features', ctypes.c_int32),
                ('save', ctypes.c_int32)] + [
        (n, ctypes.c_void_p) for n in ('image', 'params', 'drop_scales', 'features', 'workspace')] + [
        ('workspace_bytes', ctypes.c_size_t)]


# include/nfi_segformer.h (tests/test_segformer_abi.py)
SEGFORMER_EXPORTS = {
    'nfi_segformer_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(SegformerParams)]),
    'nfi_segformer_forward': (ctypes.c_int, [ctypes.POINTER(SegformerParams), ctypes.c_void_p]),
    'nfi_segformer_backward': (ctypes.c_int, [ctypes.POINTER(SegformerParams), ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_void_p]),
}

PNP_MAX_FOCALS, PNP_RECORD_DOUBLES = 64, 9


class PnpParams(ctypes.Structure):
    """struct nfi_pnp_params (include/nfi_pnp.h)."""
    _fields_ = [(n, ctypes.c_int32) for n in ('batch', 'height', 'width', 'n_focals', 'refine')] + [
        ('coords', ctypes.c_void_p), ('coords_stride', ctypes.c_int64 * 4)] + [
        (n, ctypes.c_void_p) for n in ('mask', 'focals', 'world2cam', 'focal', 'error', 'record',
                                       'workspace')] + [
        ('workspace_bytes', ctypes.c_size_t)]


# include/nfi_pnp.h (tests/test_pnp_abi.py)
PNP_EXPORTS = {
    'nfi_pnp_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(PnpParams)]),
    'nfi_pnp_solve': (ctypes.c_int, [ctypes.POINTER(PnpParams), ctypes.c_void_p]),
}

_lib = None
_lock = threading.Lock()


class NfiError(RuntimeError):
    pass


def build(verbose=False):
    """Compiles the library in-tree (nvcc, sm_90a)."""
    script = os.path.join(_HERE, 'csrc', 'build.sh')
    res = subprocess.run(['bash', script], capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
        print(res.stderr)
    if res.returncode != 0:
        raise NfiError('building libnfi_render.so failed')
    return LIB_PATH


def load():
    """Loads libnfi_render.so; raises if it has not been built."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.isfile(LIB_PATH):
                raise NfiError(
                    'libnfi_render.so is missing (%s): run '
                    'nerf_from_image_b200/csrc/build.sh or '
                    '__graft_entry__.build(); there is no fallback path.'
                    % LIB_PATH)
            lib = ctypes.CDLL(LIB_PATH)
            lib.nfi_abi_version.restype = ctypes.c_int
            got = lib.nfi_abi_version()
            if got != ABI_VERSION:
                # also under NFI_LIB_PATH: a build with another struct layout would turn into
                # memory corruption, not an error
                raise NfiError('%s has ABI version %d, this binding needs %d: rebuild it '
                               '(nerf_from_image_b200/csrc/build.sh)' % (LIB_PATH, got, ABI_VERSION))
            for name, (restype, argtypes) in (list(EXPORTS.items()) + list(LPIPS_EXPORTS.items())
                                       + list(ENCODER_EXPORTS.items()) + list(DISC_EXPORTS.items())
                                       + list(DISC_R1_EXPORTS.items())
                                       + list(SEGFORMER_EXPORTS.items())
                                       + list(PNP_EXPORTS.items())):
                fn = getattr(lib, name, None)
                if fn is None and os.environ.get('NFI_LIB_PATH'):
                    continue  # an older build under test lacks the newer entry points
                fn = getattr(lib, name)
                fn.restype = restype
                fn.argtypes = argtypes
            _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        raise NfiError(load().nfi_last_error().decode() or 'nfi error %d' % rc)


def ptr(t):
    """A tensor's device address for the C ABI; None (NULL) for None."""
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream(dev):
    """The current CUDA stream of ``dev`` for the C ABI."""
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def take_saved(ctx, what, hint=''):
    """The state an autograd forward kept in ``ctx.state`` for its backward, handed over once: the
    workspace it holds is released when the backward returns.  ``what`` names the backward in the
    refusals; ``hint`` ends the one for ``create_graph``."""
    import torch
    if ctx.state is None:
        raise NfiError('the fused %s backward ran twice on one forward (retain_graph is not '
                       'supported: the workspace is released)' % what)
    if torch.is_grad_enabled():
        raise NfiError('the fused %s backward is not differentiable (create_graph)%s'
                       % (what, ': ' + hint if hint else ''))
    state, ctx.state = ctx.state, None
    return state


def find_saved(out, what):
    """The state kept by the fused forward behind ``out`` (the first node with one on the walk down
    ``grad_fn``'s first inputs), before its backward has run."""
    fn = out.grad_fn
    while fn is not None and getattr(fn, 'state', None) is None:
        fn = fn.next_functions[0][0] if fn.next_functions else None
    if fn is None:
        raise NfiError('no saved %s forward behind this output (or its backward has already '
                       'released the workspace)' % what)
    return fn.state


_FUSED_CLASSES = {}


def switch_class(module, forward, enabled):
    """Switches ``module`` to the class ``Fused<Base>``, its reference class ``Base`` with ``forward``
    in place of ``Base.forward`` (``enabled=False`` switches it back to ``Base``); returns the module.
    The class is made once per (``Base``, ``forward``); it keeps ``Base`` as ``_nfi_unfused_class``
    and takes the ``__module__`` of ``forward``'s module."""
    base = getattr(type(module), '_nfi_unfused_class', type(module))
    if not enabled:
        module.__class__ = base
        return module
    key = (base, forward)
    if key not in _FUSED_CLASSES:
        _FUSED_CLASSES[key] = type('Fused' + base.__name__, (base,),
                                   {'forward': forward, '_nfi_unfused_class': base,
                                    '__module__': forward.__module__})
    module.__class__ = _FUSED_CLASSES[key]
    return module
