"""include/nfi_pnp.h against its ctypes table (_lib.PNP_EXPORTS, _lib.PnpParams) and the built
library, without a GPU."""
import ctypes
import os

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'nfi_pnp.h')


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    names = Hh.header_functions(_src())
    assert sorted(names) == sorted(_lib.PNP_EXPORTS)
    lib = _lib.load()
    for name in names:
        assert getattr(lib, name).restype == _lib.PNP_EXPORTS[name][0]


def test_struct_layout_matches_the_header():
    src = _src()
    assert Hh.struct_fields(src, 'nfi_pnp_params') == [f[0] for f in _lib.PnpParams._fields_]
    assert '#define NFI_PNP_MAX_FOCALS %d' % _lib.PNP_MAX_FOCALS in src
    assert '#define NFI_PNP_RECORD_DOUBLES %d' % _lib.PNP_RECORD_DOUBLES in src


def _params(b=2, h=16, w=16, f=3, refine=1):
    p = _lib.PnpParams()
    p.batch, p.height, p.width, p.n_focals, p.refine = b, h, w, f, refine
    return p


def test_workspace_and_refusals_without_a_gpu():
    lib = _lib.load()
    size = lambda p: lib.nfi_pnp_workspace_bytes(ctypes.byref(p))
    # points (5 doubles per pixel), candidates (9 doubles each), counts, each 256-aligned
    assert size(_params()) == 2 * 256 * 40 + 512 + 256
    assert lib.nfi_pnp_workspace_bytes(None) == 0
    for bad in (_params(b=0), _params(h=0), _params(f=0), _params(f=65), _params(refine=2)):
        assert size(bad) == 0
        assert len(lib.nfi_last_error()) > 0
    assert lib.nfi_pnp_solve(ctypes.byref(_params()), None) != 0   # pointers missing
    assert b'must be given' in lib.nfi_last_error()
    assert lib.nfi_pnp_solve(None, None) != 0
