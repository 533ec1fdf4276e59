"""include/nfi_lpips.h against its ctypes table (_lib.LPIPS_EXPORTS, _lib.LpipsParams) and the built
library, without a GPU.  (The other headers and _lib.EXPORTS are checked by tests/test_abi.py.)"""
import ctypes
import os

import pytest

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_lpips.h')


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    names = Hh.header_functions(_src())
    assert len(names) == 4
    assert sorted(names) == sorted(_lib.LPIPS_EXPORTS)
    assert not set(names) & set(_lib.EXPORTS)


def test_library_exports_the_lpips_symbols():
    lib = _lib.load()
    for name in _lib.LPIPS_EXPORTS:
        assert hasattr(lib, name), name
        assert getattr(lib, name).restype == _lib.LPIPS_EXPORTS[name][0]


def test_struct_layout_matches_the_header():
    src = _src()
    assert '#define NFI_LPIPS_CONVS %d' % _lib.LPIPS_CONVS in src
    assert '#define NFI_LPIPS_TAPS %d' % _lib.LPIPS_TAPS in src
    assert Hh.struct_fields(src, 'nfi_lpips_params') == [f[0] for f in _lib.LpipsParams._fields_]


def _params(n=2, h=32, w=32, save=1):
    p = _lib.LpipsParams()
    p.n, p.height, p.width, p.save = n, h, w, save
    return p


def test_workspace_sizes_and_refusals_without_a_gpu():
    lib = _lib.load()
    assert lib.nfi_lpips_workspace_bytes(None) == 0
    assert lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(h=40))) == 0    # not a multiple of 16
    assert lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(n=0))) == 0
    saved = lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(save=1)))
    plain = lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(save=0)))
    assert saved > plain > 0
    # grows linearly in N (no hidden per-call cap)
    assert lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(n=4, save=0))) > plain
    for bad in (_params(h=24), _params(n=0), _params()):   # the last one: pointers missing
        assert lib.nfi_lpips_forward(ctypes.byref(bad), None) != 0
        assert len(lib.nfi_last_error()) > 0
    assert lib.nfi_lpips_backward(ctypes.byref(_params(save=0)), None, None, None, None) != 0
    assert b'save = 1' in lib.nfi_last_error()
    # a gradient to in1 needs the save = 2 workspace
    assert lib.nfi_lpips_backward(ctypes.byref(_params(save=1)), None, None, ctypes.c_void_p(16),
                                  None) != 0
    assert b'save = 2' in lib.nfi_last_error()
    assert lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(save=2))) > saved
    assert lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(save=3))) == 0
    assert lib.nfi_lpips_saved_preactivation(ctypes.byref(_params()), 13, None, None) != 0


# Exact workspace totals: the forward, the backward and saved_preactivation walk one layout, so a
# buffer lost, taken twice or resized changes a total.  (N, H = W, save) -> bytes.
WORKSPACE_TOTALS = {
    (1, 16, 0): 59361280, (1, 16, 1): 118683648, (1, 16, 2): 118880256,
    (1, 128, 0): 92392448, (1, 128, 1): 182422528, (1, 128, 2): 195005440,
    (256, 16, 0): 193061888, (256, 16, 1): 376677376, (256, 16, 2): 427009024,
    (256, 128, 0): 8649119744, (256, 128, 1): 16693909504, (256, 128, 2): 19915134976,
}


@pytest.mark.parametrize('n, hw, save', sorted(WORKSPACE_TOTALS))
def test_workspace_keeps_its_totals(n, hw, save):
    lib = _lib.load()
    got = lib.nfi_lpips_workspace_bytes(ctypes.byref(_params(n=n, h=hw, w=hw, save=save)))
    assert got == WORKSPACE_TOTALS[(n, hw, save)]
