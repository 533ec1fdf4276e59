"""include/nfi_disc_r1.h against its ctypes table (_lib.DISC_R1_EXPORTS, _lib.DiscHvp) and the built
library, without a GPU: the functions, the hvp struct's layout, the scratch sizes and the refusals."""
import ctypes
import os

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_disc_r1.h')


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    src = _src()
    names = Hh.header_functions(src)
    assert sorted(names) == sorted(_lib.DISC_R1_EXPORTS)
    assert not set(names) & (set(_lib.EXPORTS) | set(_lib.LPIPS_EXPORTS) | set(_lib.ENCODER_EXPORTS)
                             | set(_lib.DISC_EXPORTS))
    assert '#include "nfi_disc.h"' in src


def test_library_exports_the_r1_symbols():
    lib = _lib.load()
    for name in _lib.DISC_R1_EXPORTS:
        assert hasattr(lib, name), name
        assert getattr(lib, name).restype == _lib.DISC_R1_EXPORTS[name][0]
    assert lib.nfi_abi_version() == 6


def test_hvp_struct_layout_matches_the_header():
    assert Hh.struct_fields(_src(), 'nfi_disc_hvp') == [f[0] for f in _lib.DiscHvp._fields_]
    assert ctypes.sizeof(_lib.DiscHvp) == 7 * 8


def _params(b=4, r=128, nc=4, cmap=512, save=1):
    p = _lib.DiscParams()
    p.batch, p.resolution, p.img_channels, p.cmap_dim, p.save = b, r, nc, cmap, save
    return p


def test_scratch_sizes_and_refusals_without_a_gpu():
    lib = _lib.load()
    size = lambda p: lib.nfi_disc_r1_scratch_bytes(ctypes.byref(p))
    assert lib.nfi_disc_r1_scratch_bytes(None) == 0
    for bad in (_params(b=0), _params(b=6), _params(r=96), _params(r=4), _params(r=512), _params(nc=0),
                _params(nc=5), _params(cmap=13), _params(save=2)):
        assert size(bad) == 0
    full = size(_params())
    assert full > 0
    assert size(_params(b=8)) > full                  # grows with B
    assert size(_params(r=64)) < full
    # the stacked [g; g-dot] buffers alone are larger than the forward's own activations
    assert full > lib.nfi_disc_workspace_bytes(ctypes.byref(_params(save=0)))
    g, h = _lib.DiscGrads(), _lib.DiscHvp()
    one = ctypes.c_void_p(16)
    h.g_logits, h.t_img, h.scratch, h.scratch_bytes = one, one, one, 1 << 40
    assert lib.nfi_disc_backward_hvp(ctypes.byref(_params(save=0)), ctypes.byref(h), ctypes.byref(g), None) != 0
    assert b'save = 1' in lib.nfi_last_error()
    assert lib.nfi_disc_backward_hvp(ctypes.byref(_params()), None, ctypes.byref(g), None) != 0
    assert lib.nfi_disc_backward_hvp(ctypes.byref(_params()), ctypes.byref(h), None, None) != 0
    for field in ('g_logits', 't_img', 'scratch'):
        hb = _lib.DiscHvp()
        hb.g_logits, hb.t_img, hb.scratch, hb.scratch_bytes = one, one, one, 1 << 40
        setattr(hb, field, None)
        assert lib.nfi_disc_backward_hvp(ctypes.byref(_params()), ctypes.byref(hb), ctypes.byref(g), None) != 0
        assert b'must be set' in lib.nfi_last_error()
    # pointers of the params missing: refused before anything runs
    assert lib.nfi_disc_backward_hvp(ctypes.byref(_params()), ctypes.byref(h), ctypes.byref(g), None) != 0
