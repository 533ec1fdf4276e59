"""The C-ABI library builds, loads and exports what include/*.h declare
(no compute calls: this file runs without a GPU)."""
import ctypes
import os
import re

from nerf_from_image_b200 import _lib
from tests import helpers as Hh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'nfi_render.h')
SYNTH_HEADER = os.path.join(ROOT, 'include', 'nfi_synth.h')
HEADS_HEADER = os.path.join(ROOT, 'include', 'nfi_heads.h')


def header_functions():
    return Hh.header_functions(open(HEADER).read() + open(SYNTH_HEADER).read() + open(HEADS_HEADER).read())


def test_header_and_binding_agree():
    names = header_functions()
    assert len(names) >= 12
    assert sorted(names) == sorted(_lib.EXPORTS)


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    for name in header_functions():
        assert hasattr(lib, name), name
    assert lib.nfi_abi_version() == _lib.ABI_VERSION
    assert ('#define NFI_ABI_VERSION %d' % _lib.ABI_VERSION) in open(HEADER).read()
    assert b'sm_90a' in lib.nfi_build_info()


def test_struct_layout_matches_header():
    """Field order / count of the ctypes mirrors vs the C structs."""
    src = open(HEADER).read() + open(SYNTH_HEADER).read() + open(HEADS_HEADER).read()
    for cname, cls in (('nfi_render_params', _lib.RenderParams),
                       ('nfi_render_grads', _lib.RenderGrads),
                       ('nfi_sample_params', _lib.SampleParams),
                       ('nfi_synth_layer', _lib.SynthLayer),
                       ('nfi_synth_params', _lib.SynthParams),
                       ('nfi_sdf_points_params', _lib.SdfPointsParams),
                       ('nfi_sdf_points_grads', _lib.SdfPointsGrads)):
        assert Hh.struct_fields(src, cname) == [f[0] for f in cls._fields_], cname


def test_errors_are_reported_without_a_gpu():
    lib = _lib.load()
    p = _lib.RenderParams()
    assert lib.nfi_render_forward(ctypes.byref(p), None) != 0
    assert len(lib.nfi_last_error()) > 0
    assert lib.nfi_render_workspace_bytes(None) == 0


def test_no_cpu_fallback():
    import pytest
    scene, cams = Hh.make_case('p3d_plain', batch=1, plane_res=8)
    with pytest.raises(_lib.NfiError):
        Hh.run_cuda(scene, cams, 8, 8, 8, None, None, device='cpu')


def test_graft_entry_build_checks_pass(monkeypatch):
    """__graft_entry__.build() minus the compile: its load / version / import checks."""
    import __graft_entry__ as entry
    monkeypatch.setattr(_lib, 'build', lambda verbose=False: _lib.LIB_PATH)
    entry.build()


def test_header_is_plain_c_and_links(tmp_path):
    """gcc -std=c99 -pedantic compiles a consumer of the header, links it against the built
    library and runs it (error paths only: no GPU needed); struct sizes / offsets printed by
    the C side equal the ctypes mirrors'."""
    import subprocess
    src = os.path.join(ROOT, 'tests', 'c', 'abi_check.c')
    exe = str(tmp_path / 'abi_check')
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Wextra', '-Werror', '-pedantic',
                    '-I', os.path.join(ROOT, 'include'), src, '-o', exe,
                    '-L', libdir, '-lnfi_render', '-Wl,-rpath,' + libdir], check=True)
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    out = res.stdout
    assert 'abi %d' % _lib.ABI_VERSION in out and 'sm_90a' in out
    sizes = re.search(r'sizeof params (\d+) grads (\d+) sample (\d+)', out).groups()
    assert [int(x) for x in sizes] == [ctypes.sizeof(_lib.RenderParams),
                                       ctypes.sizeof(_lib.RenderGrads),
                                       ctypes.sizeof(_lib.SampleParams)]
    synth = re.search(r'synth sizeof (\d+) layer (\d+) offsets ws (\d+) conv1 (\d+) planes (\d+)',
                      out).groups()
    assert [int(x) for x in synth] == [ctypes.sizeof(_lib.SynthParams), ctypes.sizeof(_lib.SynthLayer),
                                       _lib.SynthParams.ws.offset, _lib.SynthParams.conv1.offset,
                                       _lib.SynthParams.planes.offset]
    offs = re.search(r'offsets planes (\d+) workspace (\d+) noise_seed (\d+) points (\d+)', out).groups()
    assert [int(x) for x in offs] == [_lib.RenderParams.planes.offset,
                                      _lib.RenderParams.workspace.offset,
                                      _lib.RenderParams.noise_seed.offset,
                                      _lib.SampleParams.points.offset]


def test_backward_workspace_constant_matches_the_header():
    """fused.py sizes the backward workspace (weight images + one accumulator row buffer per CTA of
    render_wgrad_pipe) with _lib.BACKWARD_WORKSPACE_BYTES = NFI_BACKWARD_WORKSPACE_BYTES."""
    import re
    from nerf_from_image_b200 import _lib
    m = re.search(r'#define NFI_BACKWARD_WORKSPACE_BYTES \((\d+) \+ (\d+) \* (\d+)\)', open(HEADER).read())
    assert m, 'NFI_BACKWARD_WORKSPACE_BYTES missing from the header'
    a, b, c = (int(x) for x in m.groups())
    assert a + b * c == _lib.BACKWARD_WORKSPACE_BYTES
    assert ('#define NFI_VIEW_FEATURES 32') in open(HEADER).read()
