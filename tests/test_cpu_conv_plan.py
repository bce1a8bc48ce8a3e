"""Which work-item shape the conv launcher gives each launch of the published U-Net (batch 64, 256 x 256), read without a
GPU through b200ad_unet_conv_plan.

The launcher compares MMA columns issued, items (each streams the cout tile's weights) and window bytes: 32 x 32 and
16 x 16 images take 16 x 16 tiles (4 and 1 items per image instead of 5 and 2 flat ones), 64 rows and more keep 8 x 32
tiles (folded upsamples there stay flat), 8 x 8 images are packed two per item, and B200AD_CONV_DBG=4096 forces flat
items everywhere but the packed level.
"""
import ctypes as C
import os

import pytest

COLS = 12   # B200AD_CONV_PLAN_COLS
H_, W_, CIN, COUT, NSEG, UP2, PACK, TW, TH, ITEMS, AS, BS = range(COLS)


@pytest.fixture(scope="module")
def unet():
    from audio_diffusion_b200.unet import UNet2DModel
    kw = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
              down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
              up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
    return UNet2DModel(sample_size=(256, 256), **kw)


def _plan(m, dbg=None, N=64, H=256, W=256):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    old = os.environ.pop("B200AD_CONV_DBG", None)
    if dbg is not None:
        os.environ["B200AD_CONV_DBG"] = dbg
    try:
        rows = (C.c_int * (COLS * 512))()
        n = L.b200ad_unet_conv_plan(m._h, N, H, W, 132, rows, 512)
    finally:
        os.environ.pop("B200AD_CONV_DBG", None)
        if old is not None:
            os.environ["B200AD_CONV_DBG"] = old
    assert n > 0, L.b200ad_last_error().decode()
    return [tuple(rows[COLS * i:COLS * (i + 1)]) for i in range(n)]


def test_unet_item_shapes_by_level(unet):
    plan = _plan(unet)
    assert len(plan) == 101
    seen = set()
    for r in plan:
        H, W = r[H_], r[W_]
        seen.add(H)
        shape = (r[TW], r[TH])
        if H >= 64 and r[UP2]:
            assert shape == (0, 0) and not r[PACK], r
        elif H >= 64:
            assert shape == (8, 32) and not r[PACK], r
            assert r[ITEMS] == 64 * (H // 32) * (W // 8) * (r[COUT] // 128), r
        elif H in (32, 16):
            assert shape == (16, 16) and not r[PACK], r
            assert r[ITEMS] == 64 * (H // 16) * (W // 16) * (r[COUT] // 128), r
        else:
            assert H == 8 and r[PACK] == 2 and shape == (0, 0), r
            assert r[ITEMS] == 32 * (r[COUT] // 128), r
        assert 3 <= r[AS] <= 8 and 5 <= r[BS] <= 10, r
    assert seen == {256, 128, 64, 32, 16, 8}
    # the folded upsamples (four launches each, at the low-res input's size): 8 -> 16 packed, 16 -> 32 and 32 -> 64 on
    # 16 x 16 tiles, 64 -> 128 and 128 -> 256 on flat items (they do not take 8 x 32 tiles)
    ups = sorted((r[H_], r[TW], r[TH], r[PACK]) for r in plan if r[UP2])
    assert ups == sorted([(8, 0, 0, 2)] * 4 + [(16, 16, 16, 0)] * 4 + [(32, 16, 16, 0)] * 4 + [(64, 0, 0, 0)] * 4 +
                         [(128, 0, 0, 0)] * 4)


def test_unet_forced_flat(unet):
    tiled, flat = _plan(unet), _plan(unet, "4096")
    assert len(flat) == len(tiled)
    for t, f in zip(tiled, flat):
        assert (f[TW], f[TH]) == (0, 0) and f[PACK] == t[PACK], f
        H, W = f[H_], f[W_]
        if not f[PACK]:
            # flat items: 256 consecutive pixels of the padded rows (W + 1 wide)
            assert f[ITEMS] == 64 * -(-(H * (W + 1)) // 256) * (f[COUT] // 128), f


def test_flat_items_cost_more_where_tiles_fit(unet):
    """Per image and cout tile: 16 x 16 halves the items at 16 x 16 (2 -> 1) and 32 x 32 drops from 5 to 4."""
    tiled, flat = _plan(unet), _plan(unet, "4096")
    for t, f in zip(tiled, flat):
        per_t, per_f = t[ITEMS] // (64 * t[COUT] // 128), f[ITEMS] // (64 * f[COUT] // 128)
        if t[H_] == 16:
            assert (per_f, per_t) == (2, 1)
        elif t[H_] == 32:
            assert (per_f, per_t) == (5, 4)
