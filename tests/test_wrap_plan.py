"""Seamless tiling, host side (no GPU needed): the periodic tile plan (td_grid_init's `wrap`), its weight canvas
(td_grid_weights) and the grid validation of the scatter / blend entries, against tests/wrap_oracle.py."""
import ctypes
import math

import numpy as np
import pytest

import wrap_oracle as wo

SWEEP = [(L, t, ov) for L in (24, 40, 64, 100, 128, 257, 512, 2048) for t in (8, 16, 33, 64, 96, 128) for ov in (0, 4, 8, 16, 48)
         if t <= L and ov <= t - 4 and math.ceil(L / (t - ov)) <= 256]   # TD_MAX_GRID_DIM tiles per axis


def _grid(w, h, tw, th, ov, bs, wrap):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine.make_grid(w, h, tw, th, ov, bs, wrap=wrap)


@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_Y, wo.WRAP_X | wo.WRAP_Y])
def test_periodic_origins_match_oracle(wrap):
    for (L, t, ov) in SWEEP:
        w, h = {wo.WRAP_X: (L, 256), wo.WRAP_Y: (256, L)}.get(wrap, (L, L))
        tw = th = t
        g = _grid(w, h, tw, th, ov, 4, wrap)
        plan = wo.WrapPlan(w, h, tw, th, ov, 4, wrap)
        assert list(g.xs[:g.cols]) == plan.xs, (L, t, ov, wrap)
        assert list(g.ys[:g.rows]) == plan.ys, (L, t, ov, wrap)
        assert (g.tile_w, g.tile_h, g.overlap) == (plan.tile_w, plan.tile_h, plan.overlap)
        assert (g.num_batches, g.tile_bs) == (plan.num_batches, plan.tile_bs)


@pytest.mark.parametrize("L,t,ov", SWEEP)
def test_periodic_axis_covers_and_overlaps(L, t, ov):
    g = _grid(L, 16, t, 16, ov, 3, wo.WRAP_X)
    xs = list(g.xs[:g.cols])
    t = g.tile_w
    assert all(0 <= x < L for x in xs) and xs == sorted(xs) and len(set(xs)) == len(xs)
    cover = np.zeros(L, dtype=np.int64)
    for x in xs:
        cover[(x + np.arange(t)) % L] += 1
    assert cover.min() >= 1, "a pixel is not covered"
    if len(xs) > 1:
        for k in range(len(xs)):   # cyclic neighbours, the last and the first included
            gap = (xs[(k + 1) % len(xs)] - xs[k]) % L
            assert t - gap >= g.overlap, (L, t, ov, k, xs)


def test_cfg2_and_panorama_shapes():
    g = _grid(512, 512, 96, 96, 48, 4, wo.WRAP_X | wo.WRAP_Y)
    assert (g.rows, g.cols, g.num_tiles) == (11, 11, 121)
    g = _grid(2048, 512, 96, 96, 48, 4, wo.WRAP_X)
    assert g.cols == 43 and list(g.ys[:g.rows]) == wo.linear_origins(512, 96, 48)
    g = _grid(64, 40, 64, 40, 8, 2, wo.WRAP_X | wo.WRAP_Y)     # tile == canvas: one tile at the origin
    assert (g.rows, g.cols, g.xs[0], g.ys[0]) == (1, 1, 0, 0)


@pytest.mark.parametrize("w,h,tw,th,ov,bs", [(64, 48, 16, 16, 8, 4), (128, 128, 96, 96, 48, 4), (100, 37, 33, 20, 8, 3),
                                             (512, 512, 96, 96, 48, 8), (40, 40, 64, 64, 16, 1)])
def test_grid_init_wrap_zero_is_the_bounded_plan(w, h, tw, th, ov, bs):
    """wrap = 0 is the reference's bounded plan: clamps, origins, batches and the weight canvas bit for bit."""
    from oracle import tiling
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid, lib
    g = TdGrid()
    plan = tiling.GridPlan(w, h, tw, th, ov, bs, False)
    assert lib.td_grid_init(ctypes.byref(g), w, h, tw, th, ov, bs, 0) == plan.num_tiles
    assert g.wrap == 0
    assert not any(g.xs[g.cols:]) and not any(g.ys[g.rows:])      # the rest of the struct is zero, as before
    assert (g.tile_w, g.tile_h, g.overlap, g.num_batches, g.tile_bs) == (plan.tile_w, plan.tile_h, plan.overlap, plan.num_batches,
                                                                        plan.tile_bs)
    assert engine.grid_bboxes_xywh(g).tolist() == [list(b) for b in plan.bboxes]
    assert engine.grid_weights(g).view(np.uint32).tolist() == plan.weights.view(np.uint32).tolist()


@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_Y, wo.WRAP_X | wo.WRAP_Y])
@pytest.mark.parametrize("gaussian", [False, True])
@pytest.mark.parametrize("shape", [(64, 48, 16, 16, 8), (100, 37, 33, 20, 8), (96, 96, 40, 24, 12)])
def test_weights_bit_equal(wrap, gaussian, shape):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    w, h, tw, th, ov = shape
    g = _grid(w, h, tw, th, ov, 4, wrap)
    plan = wo.WrapPlan(w, h, tw, th, ov, 4, wrap, gaussian)
    got = engine.grid_weights(g, plan.tile_weights)
    assert got.dtype == np.float32 and got.view(np.uint32).tolist() == plan.weights.view(np.uint32).tolist()
    assert got.min() > 0


def test_grid_weights_rejects_a_tile_past_a_bounded_edge():
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, lib
    g = _grid(64, 48, 16, 16, 8, 4, wo.WRAP_X)
    assert g.xs[g.cols - 1] + g.tile_w > 64          # the periodic plan runs past the right edge
    g.wrap = wo.WRAP_Y                               # ... which is now bounded
    out = np.empty((48, 64), dtype=np.float32)
    st = lib.td_grid_weights(ctypes.byref(g), None, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert st == TD_ERR_INVALID_ARG


def test_bounded_grid_leaving_the_canvas_is_refused_before_launch():
    """The entries validate the plan on the host: a bounded plan whose hand-edited origins put a tile past the canvas
    returns TD_ERR_INVALID_ARG before anything is written (the weight canvas) or touches the device (the pointers here are
    never dereferenced)."""
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, TD_F16, lib
    fake = ctypes.c_void_p(256)
    for axis in ("xs", "ys"):
        g = _grid(64, 48, 16, 16, 8, 4, 0)
        origins = getattr(g, axis)
        n = g.cols if axis == "xs" else g.rows
        origins[n - 1] += 1                          # the last tile column / row now ends one pixel past the edge
        out = np.zeros((48, 64), dtype=np.float32)
        st = lib.td_grid_weights(ctypes.byref(g), None, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
        assert st == TD_ERR_INVALID_ARG and not out.any()
        st = lib.td_scatter_tiles(ctypes.byref(g), fake, fake, 2, 4, TD_F16, 0, g.num_tiles, 0, None)
        assert st == TD_ERR_INVALID_ARG and b"leaves the" in lib.td_last_error()
        ptrs = (ctypes.c_void_p * g.num_batches)(*([256] * g.num_batches))
        st = lib.td_blend_multidiffusion(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, None, fake, None, 0,
                                         None)
        assert st == TD_ERR_INVALID_ARG
        st = lib.td_blend_mixture(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, fake, fake, 0, None)
        assert st == TD_ERR_INVALID_ARG


def test_wrapped_plan_refuses_the_opt_in_forms():
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import (TD_ERR_UNSUPPORTED, TD_F16, TD_FLAG_ROWS, TD_FLAG_STRIP, TD_FLAG_TMA,
                                                                      TD_FLAG_PIPELINE, lib)
    g = _grid(64, 48, 16, 16, 8, 4, wo.WRAP_X)
    fake = ctypes.c_void_p(256)
    ptrs = (ctypes.c_void_p * g.num_batches)(*([256] * g.num_batches))
    for f in (TD_FLAG_ROWS, TD_FLAG_STRIP, TD_FLAG_TMA, TD_FLAG_PIPELINE):
        assert lib.td_scatter_tiles(ctypes.byref(g), fake, fake, 2, 4, TD_F16, 0, g.num_tiles, f, None) == TD_ERR_UNSUPPORTED
        assert lib.td_blend_multidiffusion(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, None, fake, None, f,
                                           None) == TD_ERR_UNSUPPORTED
        assert lib.td_blend_mixture(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, fake, fake, f,
                                    None) == TD_ERR_UNSUPPORTED
    assert lib.td_blend_multidiffusion_peer(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, fake, None, fake, 1,
                                            fake, 0, None) == TD_ERR_UNSUPPORTED
    assert lib.td_blend_multidiffusion_rows(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, 2, 4, TD_F16, TD_F16, fake, None, fake, None, 0,
                                            48, None, 0, None, 0, 0, 0, None) == TD_ERR_UNSUPPORTED


def test_plan_records_its_wrap_bits():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    g = engine.make_grid(64, 48, 16, 16, 8, 4, wrap=engine.WRAP_X)
    assert g.wrap == engine.WRAP_X
    assert engine.scaled_grid(g, 8).wrap == engine.WRAP_X
    assert engine.make_grid(64, 48, 16, 16, 8, 4).wrap == 0


# ------------------------------------------------------------------------------------------------ tiled VAE split
def _vae_split(h, w, tile, is_dec, wrap):
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    hook = tilevae.VAEHook.__new__(tilevae.VAEHook)
    hook.tile_size, hook.is_decoder, hook.pad = tile, is_dec, 11 if is_dec else 32
    hook.wrap_x, hook.wrap_y = bool(wrap & wo.WRAP_X), bool(wrap & wo.WRAP_Y)
    return hook.split_tiles(h, w), hook.pad


VAE_SPLITS = [(40, 52, 16, True), (1024, 1024, 96, True), (17, 130, 64, True), (200, 264, 64, False), (97, 333, 64, False),
              (512, 768, 256, False), (64, 64, 64, False)]


@pytest.mark.parametrize("h,w,tile,is_dec", VAE_SPLITS)
@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_Y, wo.WRAP_X | wo.WRAP_Y])
def test_vae_split_wrap(h, w, tile, is_dec, wrap):
    from oracle import vae as ovae
    (ib, ob), pad = _vae_split(h, w, tile, is_dec, wrap)
    assert (ib, ob) == wo.vae_split_wrap(h, w, tile, pad, is_dec, wrap)
    oh, ow = (h * 8, w * 8) if is_dec else (h // 8, w // 8)
    cover = np.zeros((oh, ow), dtype=np.int64)          # output bboxes partition the canvas
    for b in ob:
        cover[b[2]:b[3], b[0]:b[1]] += 1
    assert cover.min() == 1 and cover.max() == 1
    unscale = (lambda v: v // 8) if is_dec else (lambda v: v * 8)
    ref_ib, ref_ob = ovae.split_tiles(h, w, tile, pad, is_dec)
    for i, (bi, bo) in enumerate(zip(ib, ob)):
        for axis, bit, L in ((0, wo.WRAP_X, w), (2, wo.WRAP_Y, h)):
            lo, hi = unscale(bo[axis]), unscale(bo[axis + 1])
            if wrap & bit:
                end = L if bo[axis + 1] == (L * 8 if is_dec else L // 8) else hi       # the last cut is L itself
                assert (bi[axis], bi[axis + 1]) == (lo - pad, end + pad)                 # input = output +- pad
                if not is_dec:
                    assert bi[axis] + pad == 0 or (bi[axis] + pad) % 8 == 0                                 # encoder cuts on 8
                assert 0 <= bo[axis] < bo[axis + 1]
    # a non-wrapped axis is split exactly as td_vae_split_tiles splits it
    ref_x = sorted({(b[0], b[1], o[0], o[1]) for b, o in zip(ref_ib, ref_ob)})
    ref_y = sorted({(b[2], b[3], o[2], o[3]) for b, o in zip(ref_ib, ref_ob)})
    if not wrap & wo.WRAP_X:
        assert sorted({(b[0], b[1], o[0], o[1]) for b, o in zip(ib, ob)}) == ref_x
    if not wrap & wo.WRAP_Y:
        assert sorted({(b[2], b[3], o[2], o[3]) for b, o in zip(ib, ob)}) == ref_y


@pytest.mark.parametrize("h,w,tile,is_dec", VAE_SPLITS)
def test_vae_split_without_wrap_is_unchanged(h, w, tile, is_dec):
    from oracle import vae as ovae
    (ib, ob), pad = _vae_split(h, w, tile, is_dec, 0)
    assert (ib, ob) == tuple(map(list, ovae.split_tiles(h, w, tile, pad, is_dec)))
