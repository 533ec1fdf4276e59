"""include/nfi_segformer.h against its ctypes table (_lib.SEGFORMER_EXPORTS, _lib.SegformerParams)
and the built library, without a GPU."""
import ctypes
import os

import pytest

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_segformer.h')
B5 = (3, 6, 40, 3)


def _src():
    return open(HEADER).read()


def test_header_and_table_agree():
    names = Hh.header_functions(_src())
    assert sorted(names) == sorted(_lib.SEGFORMER_EXPORTS)
    assert not set(names) & (set(_lib.EXPORTS) | set(_lib.ENCODER_EXPORTS) | set(_lib.DISC_EXPORTS))
    lib = _lib.load()
    for name in names:
        assert getattr(lib, name).restype == _lib.SEGFORMER_EXPORTS[name][0]


def test_struct_layout_matches_the_header():
    src = _src()
    assert Hh.struct_fields(src, 'nfi_segformer_params') == [f[0] for f in _lib.SegformerParams._fields_]
    for name, value in (('STAGES', _lib.SEGFORMER_STAGES), ('MAX_DEPTH', _lib.SEGFORMER_MAX_DEPTH),
                        ('DECODER', _lib.SEGFORMER_DECODER)):
        assert '#define NFI_SEGFORMER_%s %d' % (name, value) in src


def _params(b=2, h=128, w=None, depths=B5, out=512, save=1):
    p = _lib.SegformerParams()
    p.batch, p.height, p.width = b, h, h if w is None else w
    p.depths[:] = list(depths)
    p.out_features, p.save = out, save
    return p


def test_refusals_without_a_gpu():
    lib = _lib.load()
    size = lambda p: lib.nfi_segformer_workspace_bytes(ctypes.byref(p))
    assert lib.nfi_segformer_workspace_bytes(None) == 0
    for bad in (_params(b=0), _params(h=96, w=128), _params(h=48), _params(h=288), _params(h=16),
                _params(out=96), _params(out=0), _params(depths=(3, 0, 40, 3)), _params(depths=(3, 6, 65, 3)),
                _params(save=2)):
        assert size(bad) == 0
    for bad in (_params(b=0), _params()):   # the last one: pointers missing
        assert lib.nfi_segformer_forward(ctypes.byref(bad), None) != 0
        assert len(lib.nfi_last_error()) > 0
    grads = (ctypes.c_void_p * 1064)()
    assert lib.nfi_segformer_backward(ctypes.byref(_params(save=0)), ctypes.c_void_p(16), grads, None) != 0
    assert b'save = 1' in lib.nfi_last_error()
    assert lib.nfi_segformer_backward(ctypes.byref(_params()), None, grads, None) != 0
    assert lib.nfi_segformer_backward(None, None, None, None) != 0


# Exact workspace totals at encoder-training size (128^2, B5's depths, 512 outputs): the forward and
# the backward walk one layout, so a buffer lost, taken twice or resized changes a total.
# (B, save) -> bytes.
WORKSPACE_TOTALS = {(2, 0): 62863360, (2, 1): 551391232, (32, 0): 790148096, (32, 1): 4477031424}


@pytest.mark.parametrize('key', sorted(WORKSPACE_TOTALS))
def test_workspace_totals(key):
    b, save = key
    lib = _lib.load()
    assert lib.nfi_segformer_workspace_bytes(ctypes.byref(_params(b=b, save=save))) == WORKSPACE_TOTALS[key]
