"""The discriminator's three sizers, pinned to exact totals.  The forward's workspace and the R1
scratch lay out their reverse-walk buffers through one helper (one copy of the B images for the
first-order backward inside a save = 1 workspace, two stacked copies in the scratch) from one set
of per-block maxima; offsets inside a buffer may move, but a buffer lost or taken twice changes a
total.  The sizers only lay the network out (no kernel runs), so this needs no GPU."""
import ctypes

import pytest

# (batch, resolution, img_channels, cmap_dim, [workspace save 0, workspace save 1, R1 scratch] bytes)
CASES = [
    (4, 8, 1, 0, [32315392, 74018816, 67710976]),
    (4, 64, 3, 512, [206746624, 416225280, 589748224]),
    (8, 64, 4, 0, [384096256, 755064832, 1111564288]),
    (8, 128, 3, 0, [992303104, 1783480320, 2559401984]),
    (32, 128, 4, 512, [3881129984, 6903291904, 10035339264]),
    (4, 256, 3, 512, [1083380736, 1873240064, 2625570816]),
    (32, 256, 4, 512, [8461375488, 14446796800, 20531617792]),
    # B = 6: not a multiple of the minibatch-std group of 4, so every sizer refuses it
    (6, 64, 3, 512, [0, 0, 0]),
]


@pytest.mark.parametrize('batch, res, nc, cmap_dim, want', CASES,
                         ids=['8px-b4', '64px-b4-cond', '64px-b8', '128px-b8', '128px-b32-cond',
                              '256px-b4-cond', '256px-b32-cond', 'refused'])
def test_sizers_keep_their_totals(batch, res, nc, cmap_dim, want):
    from nerf_from_image_b200 import _lib
    lib = _lib.load()

    def params(save):
        p = _lib.DiscParams()
        p.batch, p.resolution, p.img_channels, p.cmap_dim, p.save = batch, res, nc, cmap_dim, save
        return ctypes.byref(p)

    assert [lib.nfi_disc_workspace_bytes(params(0)), lib.nfi_disc_workspace_bytes(params(1)),
            lib.nfi_disc_r1_scratch_bytes(params(1))] == want
