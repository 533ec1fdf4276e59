"""Which kernels a render request reaches (csrc/nfi_route.h), pinned without a GPU: the routing
policy compiled on the CPU by tests/c/route_check.cpp, and the workspace sizes the library asks
for.  Each row of the tables names the condition that decides it."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'nerf_from_image_b200', 'csrc')

TC_3XTF32, TC_PIPE, SIMT = 'mode=2', 'mode=4', 'mode=1'
TC_MODE_REFUSAL = 'refused: tensor-core modes need S <= 128 and S % 4 == 0'
PEERS_REFUSAL = 'refused: peer outputs (n_peers > 0) need the pipelined kernel'
VIEW_GRAD_REFUSAL = 'refused: grad_view_features / grad_w3 / grad_b3 need params->view_features'

# (request, route, deciding condition).  Defaults: NFI_MLP_AUTO, S = 64, fine sampling with
# z_fine, A = 10, no extra output, a workspace of NFI_BACKWARD_WORKSPACE_BYTES.
FORWARD = [
    ('', 'pipe', 'AUTO inside the envelope'),
    ('S=128', 'pipe', 'S <= 128 and S % 4 == 0'),
    ('S=130', 'simt', 'S % 4 != 0: AUTO falls back'),
    ('S=132', 'simt', 'S > 128: AUTO falls back'),
    (TC_PIPE, 'pipe', 'an explicit tensor-core mode inside the envelope'),
    (TC_PIPE + ' S=132', TC_MODE_REFUSAL, 'explicit tensor-core mode outside the envelope'),
    (TC_3XTF32 + ' S=130', TC_MODE_REFUSAL, 'NFI_MLP_TC_3XTF32 is an alias of TC_PIPE'),
    (SIMT, 'simt', 'NFI_MLP_FP32_SIMT'),
    ('mode=5', 'simt', 'not a tensor-core mode, not refused'),
    ('extra=2 A=3', 'simt', 'semantics with NOUT_PAD = 4 stay on the SIMT kernel'),
    (TC_PIPE + ' extra=2 A=3', TC_MODE_REFUSAL, 'semantics with A <= 3 in a tensor-core mode'),
    ('extra=2 A=10', 'pipe', 'semantics with A > 3'),
    ('extra=1 A=3', 'pipe', 'coords take any palette'),
    ('normals=1', 'pipe+normals', 'normals with the fine depths saved'),
    ('normals=1 zfine=0', 'simt', 'normals without z_fine under fine sampling'),
    ('normals=1 fine=0 zfine=0', 'pipe+normals', 'no fine sampling: no fine depths needed'),
    ('normals=1 peers=2', PEERS_REFUSAL, 'normals with peers take the SIMT kernel, which has no peers'),
    ('normals=1 zfine=0 dbg=0x1000', 'pipe', 'bit 0x1000: p.normals is the phase-timer buffer'),
    ('peers=2', 'pipe', 'peers on the pipelined kernel'),
    (SIMT + ' peers=1', PEERS_REFUSAL, 'peers without the pipelined kernel'),
    ('view=1', 'pipe_vd', 'a view inside the envelope'),
    ('view=1 ' + SIMT, 'simt_vd', 'a view in NFI_MLP_FP32_SIMT'),
    ('view=1 S=132', 'simt_vd', 'a view outside the envelope under AUTO'),
    ('view=1 normals=1', 'pipe_vd+normals', 'normals after a view render'),
]

BACKWARD = [
    ('grads=planes', 'pipe', 'frozen decoder inside the envelope'),
    ('grads=planes,origins,dirs', 'pipe', 'frozen decoder, pose gradient'),
    ('grads=planes S=128', 'pipe', 'S <= 128 and S % 4 == 0'),
    ('grads=planes S=130', 'simt', 'S % 4 != 0'),
    ('grads=planes S=132', 'simt', 'S > 128'),
    ('grads=planes S=132 ' + TC_PIPE, 'simt', 'the backward falls back instead of refusing'),
    ('grads=planes ' + SIMT, 'simt', 'NFI_MLP_FP32_SIMT'),
    ('grads=planes mode=5', 'pipe', 'the backward takes any mode but FP32_SIMT'),
    ('grads=planes extra=2 A=10', 'simt', 'no semantics output on the pipelined backward'),
    ('grads=planes extra=2 A=3', 'simt', 'no semantics output on the pipelined backward'),
    ('grads=planes,extra extra=1', 'pipe', 'a coords gradient with a frozen decoder'),
    ('grads=planes ws=65536', 'pipe', 'the two weight images fit'),
    ('grads=planes ws=65535', 'simt', 'no room for the two weight images'),
    ('grads=planes ws=0', 'simt', 'no workspace'),
    ('grads=planes,w1', 'wgrad_planes', 'decoder gradients, planes, no pose: one sweep'),
    ('grads=palette,w2', 'wgrad_planes', 'any non-decoder gradient but the pose: one sweep'),
    ('grads=planes,w1,origins,dirs', 'pipe+wgrad', 'a pose gradient: two kernels'),
    ('grads=w1,b1,w2,b2', 'wgrad', 'decoder gradients alone'),
    ('grads=planes,w1 dbg=0x2000', 'pipe+wgrad', 'bit 0x2000: two sweeps anyway'),
    ('grads=planes,w1,extra extra=1', 'simt', 'a coords gradient with decoder gradients'),
    ('grads=planes,w1 ws=65536', 'simt', 'no room for the accumulator rows'),
    ('grads=planes,w1 ws=5308415', 'simt', 'one byte short of NFI_BACKWARD_WORKSPACE_BYTES'),
    ('grads=planes,w1 ' + SIMT, 'simt', 'NFI_MLP_FP32_SIMT'),
    ('grads=planes view=1 ws=98304', 'pipe_vd', 'a view, decoder and mapper frozen'),
    ('grads=planes,view,origins,dirs view=1 ws=98304', 'pipe_vd', 'view features and pose'),
    ('grads=planes view=1 ws=98303', 'simt_vd', 'no room for the two view weight images'),
    ('grads=planes view=1 S=132', 'simt_vd', 'a view outside the envelope'),
    ('grads=planes view=1 ' + SIMT, 'simt_vd', 'a view in NFI_MLP_FP32_SIMT'),
    ('grads=planes,w1 view=1', 'simt_vd', 'a view with a decoder gradient'),
    ('grads=planes,w3 view=1', 'simt_vd', 'a view with a W3 gradient'),
    ('grads=planes,b3 view=1', 'simt_vd', 'a view with a b3 gradient'),
    ('grads=planes,view', VIEW_GRAD_REFUSAL, 'grad_view_features without a view'),
    ('grads=planes,w3', VIEW_GRAD_REFUSAL, 'grad_w3 without a view'),
    ('grads=planes,b3 ' + SIMT, VIEW_GRAD_REFUSAL, 'grad_b3 without a view, in any mode'),
]


@pytest.fixture(scope='module')
def route_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('route') / 'route_check')
    subprocess.run(['g++', '-std=c++17', '-O1', '-Wall', '-Wextra', '-Werror', '-I', CSRC,
                    '-I', os.path.join(ROOT, 'include'),
                    os.path.join(ROOT, 'tests', 'c', 'route_check.cpp'), '-o', exe], check=True)
    return exe


def _routes(exe, lines):
    out = subprocess.run([exe], input='\n'.join(lines) + '\n', capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(lines)
    return out


@pytest.mark.parametrize('request_, want, why', FORWARD, ids=[r[0] or 'default' for r in FORWARD])
def test_forward_route(route_check, request_, want, why):
    got, = _routes(route_check, ['fwd ' + request_])
    assert got.startswith(want) and (want.startswith('refused') or got == want), why


@pytest.mark.parametrize('request_, want, why', BACKWARD, ids=[r[0] for r in BACKWARD])
def test_backward_route(route_check, request_, want, why):
    got, = _routes(route_check, ['bwd ' + request_])
    assert got.startswith(want) and (want.startswith('refused') or got == want), why


# (fields of nfi_render_params, bytes nfi_render_workspace_bytes returned before the routing moved
# into nfi_route.h).  32 images of 128 x 128 rays are 4096 tiles: the persistent kernels are capped
# at 160 CTAs, the SIMT kernel takes one slab per tile.
TRAINING = dict(batch=32, height=128, width=128, num_samples=64, fine_sampling=1, n_attention=10,
                use_sdf=1)
WORKSPACE = [
    (dict(TRAINING), 36733184),
    (dict(TRAINING, fine_sampling=0), 33024),
    (dict(TRAINING, compute_normals=1, z_fine=1), 36765952),
    (dict(TRAINING, extra_mode=2), 94404864),
    (dict(TRAINING, extra_mode=2, n_attention=3), 1073774848),
    (dict(TRAINING, view_features=1), 36765952),
    (dict(TRAINING, num_samples=132), 1384153344),
    (dict(TRAINING, mlp_mode=1, compute_normals=1), 1073774848),
    (dict(TRAINING, batch=1, height=64, width=64), 7373056),
]


@pytest.mark.parametrize('fields, want', WORKSPACE, ids=[str(i) for i in range(len(WORKSPACE))])
def test_workspace_bytes(fields, want):
    from nerf_from_image_b200 import _lib
    p = _lib.RenderParams()
    for k, v in fields.items():
        setattr(p, k, v)
    p.scene_range = 1.0
    assert _lib.load().nfi_render_workspace_bytes(ctypes.byref(p)) == want


def test_backward_images_constant_matches_the_layout():
    """fused.py sizes a frozen-decoder backward's workspace with _lib.BACKWARD_IMAGES_BYTES."""
    from nerf_from_image_b200 import _lib
    layout = open(os.path.join(CSRC, 'nfi_layout.h')).read()
    val = lambda name: int(re.search(r'constexpr int %s = (\d+);' % name, layout).group(1))
    assert val('kBwdImageOffset') + val('kBwdImageBytes') == _lib.BACKWARD_IMAGES_BYTES
