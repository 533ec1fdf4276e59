"""include/nfi_disc.h against its ctypes table (_lib.DISC_EXPORTS, _lib.DiscParams, _lib.DiscGrads)
and the built library, without a GPU."""
import ctypes
import os

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_disc.h')


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    names = Hh.header_functions(_src())
    assert len(names) == 4
    assert sorted(names) == sorted(_lib.DISC_EXPORTS)
    assert not set(names) & (set(_lib.EXPORTS) | set(_lib.LPIPS_EXPORTS) | set(_lib.ENCODER_EXPORTS))


def test_library_exports_the_discriminator_symbols():
    lib = _lib.load()
    for name in _lib.DISC_EXPORTS:
        assert hasattr(lib, name), name
        assert getattr(lib, name).restype == _lib.DISC_EXPORTS[name][0]


def test_struct_layouts_match_the_header():
    src = _src()
    assert '#define NFI_DISC_MAX_BLOCKS %d' % _lib.DISC_MAX_BLOCKS in src
    assert Hh.struct_fields(src, 'nfi_disc_params') == [f[0] for f in _lib.DiscParams._fields_]
    assert Hh.struct_fields(src, 'nfi_disc_grads') == [f[0] for f in _lib.DiscGrads._fields_]


def _params(b=4, r=128, nc=4, cmap=512, save=1):
    p = _lib.DiscParams()
    p.batch, p.resolution, p.img_channels, p.cmap_dim, p.save = b, r, nc, cmap, save
    return p


def test_workspace_sizes_and_refusals_without_a_gpu():
    lib = _lib.load()
    size = lambda p: lib.nfi_disc_workspace_bytes(ctypes.byref(p))
    assert lib.nfi_disc_workspace_bytes(None) == 0
    for bad in (_params(b=0), _params(b=6), _params(r=96), _params(r=4), _params(r=512), _params(nc=0),
                _params(nc=5), _params(cmap=13), _params(save=2)):
        assert size(bad) == 0
    saved, plain = size(_params(save=1)), size(_params(save=0))
    assert saved > plain > 0
    assert size(_params(b=8, save=0)) > plain                        # grows with B
    assert size(_params(r=64)) < saved
    for bad in (_params(b=0), _params()):   # the last one: pointers missing
        assert lib.nfi_disc_forward(ctypes.byref(bad), None) != 0
        assert len(lib.nfi_last_error()) > 0
    g = _lib.DiscGrads()
    one = ctypes.c_void_p(16)
    assert lib.nfi_disc_backward(ctypes.byref(_params(save=0)), one, None, None, ctypes.byref(g), None) != 0
    assert b'save = 1' in lib.nfi_last_error()
    assert lib.nfi_disc_backward(ctypes.byref(_params()), None, None, None, ctypes.byref(g), None) != 0
    assert lib.nfi_disc_backward(ctypes.byref(_params()), one, None, None, None, None) != 0
    assert lib.nfi_disc_saved_preactivation(ctypes.byref(_params()), 6, 0, one, None) != 0
    assert lib.nfi_disc_saved_preactivation(ctypes.byref(_params()), 1, 0, one, None) != 0
    assert lib.nfi_disc_saved_preactivation(ctypes.byref(_params(save=0)), 0, 1, one, None) != 0
