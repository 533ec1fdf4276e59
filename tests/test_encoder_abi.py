"""include/nfi_encoder.h against its ctypes table (_lib.ENCODER_EXPORTS, _lib.EncoderParams,
_lib.EncoderGrads) and the built library, without a GPU."""
import ctypes
import os

import pytest

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_encoder.h')


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    names = Hh.header_functions(_src())
    assert len(names) == 4
    assert sorted(names) == sorted(_lib.ENCODER_EXPORTS)
    assert not set(names) & (set(_lib.EXPORTS) | set(_lib.LPIPS_EXPORTS))


def test_library_exports_the_encoder_symbols():
    lib = _lib.load()
    for name in _lib.ENCODER_EXPORTS:
        assert hasattr(lib, name), name
        assert getattr(lib, name).restype == _lib.ENCODER_EXPORTS[name][0]


def test_struct_layouts_match_the_header():
    src = _src()
    assert '#define NFI_ENCODER_MAPS %d' % _lib.ENCODER_MAPS in src
    assert Hh.struct_fields(src, 'nfi_encoder_params') == [f[0] for f in _lib.EncoderParams._fields_]
    assert Hh.struct_fields(src, 'nfi_encoder_grads') == [f[0] for f in _lib.EncoderGrads._fields_]


def _params(b=2, h=8, w=8, c=512, pose=1, latent=1, save=1):
    p = _lib.EncoderParams()
    p.batch, p.height, p.width, p.channels = b, h, w, c
    p.pose_regressor, p.latent_regressor, p.save = pose, latent, save
    return p


def test_workspace_sizes_and_refusals_without_a_gpu():
    lib = _lib.load()
    size = lambda p: lib.nfi_encoder_workspace_bytes(ctypes.byref(p))
    assert lib.nfi_encoder_workspace_bytes(None) == 0
    for bad in (_params(b=0), _params(h=0), _params(w=2000), _params(c=96), _params(pose=0, latent=0),
                _params(save=2), _params(pose=2)):
        assert size(bad) == 0
    saved, plain = size(_params(save=1)), size(_params(save=0))
    assert saved > plain > 0
    assert size(_params(b=4, save=0)) > plain                       # grows with B
    assert size(_params(pose=0)) < saved and size(_params(latent=0)) < saved
    for bad in (_params(b=0), _params()):   # the last one: pointers missing
        assert lib.nfi_encoder_forward(ctypes.byref(bad), None) != 0
        assert len(lib.nfi_last_error()) > 0
    g = _lib.EncoderGrads()
    assert lib.nfi_encoder_backward(ctypes.byref(_params(save=0)), None, None, ctypes.byref(g), None) != 0
    assert b'save = 1' in lib.nfi_last_error()
    assert lib.nfi_encoder_backward(ctypes.byref(_params()), None, None, ctypes.byref(g), None) != 0
    assert lib.nfi_encoder_backward(ctypes.byref(_params()), None, None, None, None) != 0
    assert lib.nfi_encoder_saved_activation(ctypes.byref(_params()), 5, None, None) != 0
    assert lib.nfi_encoder_saved_activation(ctypes.byref(_params(latent=0)), 3, ctypes.c_void_p(16), None) != 0


# Exact workspace totals at the encoder-training feature size (32 x 32 x 512, 128^2 images): the
# forward, the backward and saved_activation walk one layout, so a buffer lost, taken twice or
# resized changes a total.  (B, pose head, latent head, save) -> bytes.
WORKSPACE_TOTALS = {
    (2, 1, 0, 0): 163252224, (2, 1, 0, 1): 412157952, (2, 0, 1, 0): 22021120,
    (2, 0, 1, 1): 58737664, (2, 1, 1, 0): 181078016, (2, 1, 1, 1): 439420928,
    (32, 1, 0, 0): 2302347264, (32, 1, 0, 1): 5700913152, (32, 0, 1, 0): 210764800,
    (32, 0, 1, 1): 373556224, (32, 1, 1, 0): 2446002176, (32, 1, 1, 1): 5854005248,
}


@pytest.mark.parametrize('b, pose, latent, save', sorted(WORKSPACE_TOTALS))
def test_workspace_keeps_its_totals(b, pose, latent, save):
    lib = _lib.load()
    p = _params(b=b, h=32, w=32, pose=pose, latent=latent, save=save)
    assert lib.nfi_encoder_workspace_bytes(ctypes.byref(p)) == WORKSPACE_TOTALS[(b, pose, latent, save)]
