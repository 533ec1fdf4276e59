"""ctypes binding of libnfi_render.so (the C ABI declared in include/nfi_render.h).

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
ABI_VERSION = 5  # NFI_ABI_VERSION of include/nfi_render.h
MAX_PEERS = 7
BACKWARD_WORKSPACE_BYTES = 65536 + 160 * 32768  # NFI_BACKWARD_WORKSPACE_BYTES

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


class SdfPointsParams(ctypes.Structure):
    """struct nfi_sdf_points_params (include/nfi_heads.h)."""
    _fields_ = [('batch', ctypes.c_int32), ('plane_res', ctypes.c_int32),
                ('scene_range', ctypes.c_float), ('n_points', ctypes.c_int64)] + [
        (n, ctypes.c_void_p) for n in ('planes', 'w1', 'b1', 'w2', 'b2', 'points', 'd', 'grad')]


class SdfPointsGrads(ctypes.Structure):
    """struct nfi_sdf_points_grads."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        'g_d', 'g_grad', 'grad_planes', 'grad_w1', 'grad_b1', 'grad_w2_row0', 'grad_b2_0')]


# every symbol include/*.h declare (tests/test_abi.py checks the
# header against this table and the table against the built library)
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
    'nfi_synthesis_param_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(SynthParams)]),
    'nfi_synthesis_backward_params': (ctypes.c_int, [ctypes.POINTER(SynthParams),
                                                     ctypes.POINTER(SynthGrads),
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
            for name, (restype, argtypes) in EXPORTS.items():
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
