"""The synthesis network's four sizers, pinned to exact totals.  The forward, the backward and the
HVP lay their workspaces out through shared helpers (one backward scratch for one or two stacked
copies, one weight-GEMM plan for the partials); offsets inside a workspace may move, but a buffer
lost or taken twice changes a total.  The sizers only lay the network out (no kernel runs), so this
needs no GPU."""
import ctypes

import pytest

SIZERS = ('nfi_synthesis_workspace_bytes', 'nfi_synthesis_saved_workspace_bytes',
          'nfi_synthesis_param_workspace_bytes', 'nfi_synthesis_hvp_scratch_bytes')

TEST_NET = dict(img_resolution=16, w_dim=64, num_ws=6, channels=(64, 64, 32))
# bench.py's 256^2 network: 7 blocks, min(32768 / r, 512) channels at resolution r
FULL_NET = dict(img_resolution=256, w_dim=512, num_ws=14,
                channels=tuple(min(32768 // r, 512) for r in (4, 8, 16, 32, 64, 128, 256)))

# (network, batch, [plain, saved, param, hvp] bytes)
CASES = [
    (TEST_NET, 1, [907264, 2086912, 2299904, 1640448]),
    (TEST_NET, 2, [1122304, 2867200, 3145728, 2504704]),
    (TEST_NET, 4, [1552384, 4427776, 4837376, 4233216]),
    (dict(img_resolution=32, w_dim=64, num_ws=8, channels=(128, 64, 96, 32)), 3,
     [5171200, 15825920, 17988608, 18252800]),
    (FULL_NET, 16, [3655787520, 11792770048, 13959128064, 17318183936]),
    (FULL_NET, 32, [7206241280, 23385293824, 27699135488, 34522579968]),
    # 48 channels: not a multiple of 32, so every sizer refuses the network
    (dict(TEST_NET, channels=(64, 48, 32)), 2, [0, 0, 0, 0]),
]


@pytest.mark.parametrize('net, batch, want', CASES,
                         ids=['16px-b1', '16px-b2', '16px-b4', '32px-mixed-b3', '256px-b16',
                              '256px-b32', 'refused'])
def test_sizers_keep_their_totals(net, batch, want):
    from nerf_from_image_b200 import _lib
    lib = _lib.load()
    P = _lib.SynthParams()
    P.batch, P.img_channels = batch, 96
    P.img_resolution, P.w_dim, P.num_ws = net['img_resolution'], net['w_dim'], net['num_ws']
    P.num_blocks = len(net['channels'])
    for i, c in enumerate(net['channels']):
        P.channels[i] = c
    assert [getattr(lib, name)(ctypes.byref(P)) for name in SIZERS] == want
