"""Tiled-VAE inpainting without a GPU: the active-tile rule restated in numpy on the decoder's output rectangles,
`VAEHook.set_inpaint_mask` refusals, the argument checks `td_vae_active_tiles` makes before any device work, and the tile
shard's round robin over the tiles a pass runs."""
import ctypes

import numpy as np
import pytest
import torch

from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, tilevae


def active_rule(mask: np.ndarray, rects) -> np.ndarray:
    """bool [T]: rectangle [x1, x2, y1, y2] is active when one element of mask [P, H, W] inside it, over all planes, is not
    exactly 1.0 (a NaN compares unequal)."""
    m = np.asarray(mask).reshape(-1, mask.shape[-2], mask.shape[-1])
    return np.array([bool((m[:, b[2]:b[3], b[0]:b[1]] != 1).any()) for b in rects], dtype=bool)


def decoder_rects(h, w, tile, wrap=0):
    """Output rectangles of the decoder split of a [h, w] latent (image canvas [8h, 8w])."""
    hook = tilevae.VAEHook(torch.nn.Conv2d(1, 1, 1), tile, True, fast_decoder=True, fast_encoder=True, color_fix=False)
    hook.wrap_x, hook.wrap_y = bool(wrap & 1), bool(wrap & 2)
    return hook.split_tiles(h, w)[1]


SPLITS = {"cfg4": (1024, 1024, 96, 0), "ragged": (37, 53, 8, 0), "wrap_x": (37, 53, 8, 1), "wrap_xy": (40, 52, 8, 3)}


@pytest.mark.parametrize("split", list(SPLITS))
def test_output_rectangles_partition_the_image_canvas(split):
    """Bounded and wrapped: the output rectangles are canvas rectangles and each image pixel lies in exactly one, so a
    skipped rectangle's pixels are the fill and nothing else writes them."""
    h, w, tile, wrap = SPLITS[split]
    rects = decoder_rects(h, w, tile, wrap)
    cover = np.zeros((8 * h, 8 * w), dtype=np.int32)
    for x1, x2, y1, y2 in rects:
        assert 0 <= x1 < x2 <= 8 * w and 0 <= y1 < y2 <= 8 * h, (x1, x2, y1, y2)
        cover[y1:y2, x1:x2] += 1
    assert (cover == 1).all()
    if split == "cfg4":
        assert len(rects) == 121


NOT_ONE = [np.nextafter(np.float32(1), np.float32(2)), np.nextafter(np.float32(1), np.float32(0)), 0.0, -0.0, np.inf, -np.inf,
           np.nan, -1.0]


@pytest.mark.parametrize("planes", [1, 3])
def test_one_element_at_each_edge_and_corner_flags_exactly_its_rectangle(planes):
    h, w, tile, _ = SPLITS["ragged"]
    rects = decoder_rects(h, w, tile)
    H, W = 8 * h, 8 * w
    for t, (x1, x2, y1, y2) in enumerate(rects):
        spots = [(y1, x1), (y1, x2 - 1), (y2 - 1, x1), (y2 - 1, x2 - 1), (y1, (x1 + x2) // 2), ((y1 + y2) // 2, x2 - 1)]
        for k, (y, x) in enumerate(spots):
            m = np.ones((planes, H, W), dtype=np.float32)
            m[k % planes, y, x] = NOT_ONE[k % len(NOT_ONE)]
            want = np.zeros(len(rects), dtype=bool)
            want[t] = True
            assert (active_rule(m, rects) == want).all(), (t, y, x)
    assert not active_rule(np.ones((planes, H, W), dtype=np.float32), rects).any()


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_values_next_to_one_are_not_one(dtype):
    one = dtype(1)
    for v in (np.nextafter(one, dtype(2)), np.nextafter(one, dtype(0)), dtype(0), -dtype(0), dtype(np.inf), dtype(np.nan)):
        m = np.ones((2, 16, 16), dtype=dtype)
        m[1, 15, 15] = v
        assert active_rule(m, [[0, 16, 0, 16], [0, 15, 0, 15]]).tolist() == [True, False], v


# ------------------------------------------------------------------------------------------ VAEHook.set_inpaint_mask refusals
def _hook(is_dec=True, fast=True):
    return tilevae.VAEHook(torch.nn.Conv2d(1, 1, 1), 8, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)


def _refused(hook, exc, mask, fill=None):
    before = dict(hook.__dict__)
    with pytest.raises(exc):
        hook.set_inpaint_mask(mask, fill)
    assert hook.__dict__.keys() == before.keys() and all(hook.__dict__[k] is v for k, v in before.items())


def test_encoder_and_slow_mode_are_refused():
    m = torch.ones(64, 64)
    _refused(_hook(is_dec=False), NotImplementedError, m)
    _refused(_hook(fast=False), NotImplementedError, m)
    _refused(_hook(is_dec=False, fast=False), NotImplementedError, m)


@pytest.mark.parametrize("mask", [torch.ones(64), torch.ones(2, 64, 64), torch.ones(2, 3, 64, 64), torch.ones(1, 1, 1, 64, 64),
                                  torch.ones(0, 64), torch.ones(0, 1, 64, 64), torch.ones(64, 64, dtype=torch.float64),
                                  torch.ones(64, 64, dtype=torch.int32), torch.ones(64, 64, dtype=torch.bool),
                                  np.ones((64, 64), dtype=np.float32)],
                         ids=["1d", "3d_planes", "4d_channels", "5d", "empty", "no_images", "f64", "i32", "bool", "numpy"])
def test_bad_masks_are_refused_without_a_change(mask):
    _refused(_hook(), ValueError, mask)


@pytest.mark.parametrize("fill", [torch.zeros(3, 64, 64), torch.zeros(1, 3, 64, 32), torch.zeros(1, 3, 64, 64, dtype=torch.float64),
                                  torch.zeros(1, 3, 64, 64, dtype=torch.int16), torch.zeros(0, 3, 64, 64), "zeros"],
                         ids=["3d", "size", "f64", "i16", "empty", "str"])
def test_bad_fills_are_refused_without_a_change(fill):
    _refused(_hook(), ValueError, torch.ones(1, 64, 64, dtype=torch.float16), fill)


def test_a_host_mask_or_fill_is_refused():
    _refused(_hook(), ValueError, torch.ones(64, 64))
    _refused(_hook(), ValueError, torch.ones(64, 64, dtype=torch.float16), torch.zeros(1, 3, 64, 64))


def test_refusal_keeps_a_mask_set_earlier():
    hook = _hook()
    hook.inpaint_mask = object()           # stands for a device mask set earlier (no GPU here)
    _refused(hook, ValueError, torch.ones(5, 64, 64))
    _refused(hook, ValueError, torch.ones(64, 64))


# ------------------------------------------------------------------------------------------ td_vae_active_tiles argument checks
def _call(mask=0x1000, planes=1, H=64, W=64, dtype=_cabi.TD_F16, rects=((0, 8, 0, 8),), n=None, out=0x2000):
    r = np.ascontiguousarray(np.asarray(rects, dtype=np.int32).reshape(-1, 4))
    p = r.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)) if len(r) else None
    return _cabi.lib.td_vae_active_tiles(mask, planes, H, W, dtype, p, len(r) if n is None else n, out, None)


@pytest.mark.parametrize("case", [
    dict(mask=None), dict(out=None), dict(rects=()), dict(mask=0x1001), dict(mask=0x1002, dtype=_cabi.TD_F32),
    dict(planes=0), dict(planes=-1), dict(H=0), dict(W=-3), dict(dtype=3), dict(dtype=-1), dict(n=0), dict(n=-1),
    dict(rects=((0, 0, 0, 8),)), dict(rects=((4, 3, 0, 8),)), dict(rects=((0, 8, 5, 5),)), dict(rects=((-1, 8, 0, 8),)),
    dict(rects=((0, 65, 0, 8),)), dict(rects=((0, 8, 0, 65),)), dict(rects=((0, 8, -2, 8),)),
    dict(rects=((0, 8, 0, 8), (0, 8, 0, 8), (60, 64, 60, 65))),
])
def test_active_tiles_refusals_come_before_any_device_work(case):
    """Fake device addresses: each call is refused by the host checks, so nothing reaches the device."""
    assert _call(**case) == _cabi.TD_ERR_INVALID_ARG, _cabi.lib.td_last_error()


def test_active_tiles_refuses_more_mask_rows_than_the_grid_holds():
    assert _call(planes=2 ** 16, H=2 ** 15 + 1) == _cabi.TD_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------ tile shard
def test_the_shard_round_robins_over_the_tiles_a_pass_runs():
    active = [1, 4, 5, 6, 9, 17, 30]
    for world in (1, 2, 3, 4, 8):
        shares = [tilevae.shard_tiles(active, world, r) for r in range(world)]
        assert sorted(sum(shares, [])) == active
        assert max(map(len, shares)) - min(map(len, shares)) <= 1, shares
        for r, s in enumerate(shares):
            assert s == [t for j, t in enumerate(active) if j % world == r]
    # every tile of the split: the fixed assignment of an unmasked call (tile i on rank i % world)
    assert tilevae.shard_tiles(range(10), 3, 1) == [1, 4, 7]
    assert tilevae.shard_tiles([], 2, 1) == []
