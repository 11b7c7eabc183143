"""SpotDiffusion host side (no GPU): td_grid_shift / td_grid_shift_bounds against tests/spot_oracle.py, the step-plan
invariants, the refusals, the shift schedule and the features the tile method refuses."""
import ctypes
import random
import types

import numpy as np
import pytest

import spot_oracle as so

LENGTHS = [64, 96, 97, 150, 512, 513, 2048]
PARTNER = {64: 150, 96: 97, 97: 64, 150: 96, 512: 513, 513: 512, 2048: 96}   # the other axis of the canvas
TILES = [64, 96, 128]
OVERLAPS = [0, 8, 48]
WRAPS = [0, so.WRAP_X, so.WRAP_Y, so.WRAP_X | so.WRAP_Y]


def _engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


def _shifts(lo, hi, small, rng):
    """Every allowed shift on a small canvas, else the ends and a sample."""
    if small or hi - lo <= 12:
        return list(range(lo, hi))
    return sorted({lo, hi - 1, *rng.sample(range(lo, hi), 10)})


def _check_axis(origins, L, t, periodic, n_windows):
    assert len(origins) == n_windows
    assert all(origins[k] < origins[k + 1] for k in range(len(origins) - 1)), origins
    if periodic:
        assert all(0 <= o < L for o in origins), origins
    else:
        assert all(0 <= o <= L - t for o in origins), origins
    assert so.coverage(origins, L, t, periodic).min() >= 1, "a position no window covers"


@pytest.mark.parametrize("wrap", WRAPS)
@pytest.mark.parametrize("overlap", OVERLAPS)
@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("L", LENGTHS)
def test_step_plan_matches_oracle(L, tile, overlap, wrap):
    engine = _engine()
    w, h, bs = L, PARTNER[L], 4
    g = engine.make_grid(w, h, tile, tile, overlap, bs, wrap=wrap)
    b = engine.shift_bounds(g)
    assert b == so.bounds(w, h, tile, tile, overlap, wrap)
    rng = random.Random(L * 1000 + tile * 10 + overlap + wrap)
    small = L <= 150 and PARTNER[L] <= 150
    px, py = bool(wrap & so.WRAP_X), bool(wrap & so.WRAP_Y)
    counts = set()
    xs_list = _shifts(b[0], b[1], small, rng)
    ys_list = _shifts(b[2], b[3], small, rng)
    pairs = [(sx, ys_list[i % len(ys_list)]) for i, sx in enumerate(xs_list)] + \
            [(xs_list[i % len(xs_list)], sy) for i, sy in enumerate(ys_list)]
    for sx, sy in pairs:
        s = engine.shift_grid(g, sx, sy, bs)
        plan = so.SpotPlan(w, h, tile, tile, overlap, bs, wrap, sx, sy)
        got_xs, got_ys = list(s.xs[:s.cols]), list(s.ys[:s.rows])
        assert got_xs == plan.xs and got_ys == plan.ys, (sx, sy)
        assert (s.W, s.H, s.tile_w, s.tile_h, s.overlap, s.wrap) == (g.W, g.H, g.tile_w, g.tile_h, g.overlap, g.wrap)
        assert (s.num_tiles, s.num_batches, s.tile_bs) == (len(plan.bboxes), plan.num_batches, plan.tile_bs)
        assert [tuple(int(v) for v in r) for r in engine.grid_bboxes_xywh(s)] == plan.bboxes
        _check_axis(got_xs, w, s.tile_w, px, len(plan.xs))
        _check_axis(got_ys, h, s.tile_h, py, len(plan.ys))
        counts.add((s.cols, s.rows))
        cx = engine.axis_coverage(got_xs, w, s.tile_w, px)
        cy = engine.axis_coverage(got_ys, h, s.tile_h, py)
        assert np.array_equal(cx, so.coverage(got_xs, w, s.tile_w, px)) and np.array_equal(cy, so.coverage(got_ys, h, s.tile_h, py))
        assert engine.counts_allow_fast_divide(s) == (int(cx.max()) * int(cy.max()) <= 4096)
    assert len(counts) == 1, f"the window count depends on the shift: {counts}"


def test_window_counts_of_the_issue_geometries():
    """cfg2's 512x512 latent at tile 96: 100 windows for MultiDiffusion at overlap 48, 36 at overlap 0, 49 for a bounded
    SpotDiffusion plan at overlap 0 and 36 seamless; the [512, 2048] panorama wrapped in x: 430 and 154."""
    engine = _engine()
    assert engine.make_grid(512, 512, 96, 96, 48, 1).num_tiles == 100
    assert engine.make_grid(512, 512, 96, 96, 0, 1).num_tiles == 36
    assert engine.shift_grid(engine.make_grid(512, 512, 96, 96, 0, 1), 1, 1, 1).num_tiles == 49
    assert engine.shift_grid(engine.make_grid(512, 512, 96, 96, 0, 1, wrap=3), 0, 0, 1).num_tiles == 36
    assert engine.make_grid(2048, 512, 96, 96, 48, 1, wrap=1).num_tiles == 430
    assert engine.shift_grid(engine.make_grid(2048, 512, 96, 96, 0, 1, wrap=1), 0, 1, 1).num_tiles == 154


def _sentinel():
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
    out = TdGrid()
    ctypes.memset(ctypes.addressof(out), 0x5A, ctypes.sizeof(out))
    return out, bytes(out)


@pytest.mark.parametrize("wrap", WRAPS)
def test_out_of_range_shifts_are_refused(wrap):
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    engine = _engine()
    g = engine.make_grid(150, 97, 64, 64, 8, 4, wrap=wrap)
    lo_x, hi_x, lo_y, hi_y = engine.shift_bounds(g)
    for sx, sy in [(lo_x - 1, lo_y), (hi_x, lo_y), (lo_x, lo_y - 1), (lo_x, hi_y), (-1000, 1000)]:
        out, before = _sentinel()
        st = _cabi.lib.td_grid_shift(ctypes.byref(g), sx, sy, 4, ctypes.byref(out))
        assert st == _cabi.TD_ERR_INVALID_ARG, (sx, sy)
        assert bytes(out) == before
    out, before = _sentinel()
    assert _cabi.lib.td_grid_shift(ctypes.byref(g), lo_x, lo_y, 0, ctypes.byref(out)) == _cabi.TD_ERR_INVALID_ARG
    assert _cabi.lib.td_grid_shift(None, lo_x, lo_y, 4, ctypes.byref(out)) == _cabi.TD_ERR_INVALID_ARG
    assert bytes(out) == before
    assert _cabi.lib.td_grid_shift(ctypes.byref(g), lo_x, lo_y, 4, None) == _cabi.TD_ERR_INVALID_ARG
    assert _cabi.lib.td_grid_shift_bounds(None, (ctypes.c_int32 * 4)()) == _cabi.TD_ERR_INVALID_ARG
    assert _cabi.lib.td_grid_shift_bounds(ctypes.byref(g), None) == _cabi.TD_ERR_INVALID_ARG


def test_malformed_base_plans_are_refused():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
    engine = _engine()
    good = engine.make_grid(150, 97, 64, 64, 8, 4)
    for field, value in [("cols", 0), ("rows", 257), ("wrap", 4)]:
        g = TdGrid.from_buffer_copy(good)
        setattr(g, field, value)
        out, before = _sentinel()
        assert _cabi.lib.td_grid_shift(ctypes.byref(g), 0, 0, 4, ctypes.byref(out)) == _cabi.TD_ERR_INVALID_ARG, field
        assert bytes(out) == before
    g = TdGrid.from_buffer_copy(good)
    g.xs[1], g.xs[2] = g.xs[2], g.xs[1]                   # decreasing origins
    assert _cabi.lib.td_grid_shift(ctypes.byref(g), 1, 1, 4, ctypes.byref(TdGrid())) == _cabi.TD_ERR_INVALID_ARG
    g = TdGrid.from_buffer_copy(good)
    g.xs[g.cols - 1] = g.W - g.tile_w + 1                  # a tile leaving the bounded canvas
    assert _cabi.lib.td_grid_shift(ctypes.byref(g), 1, 1, 4, ctypes.byref(TdGrid())) == _cabi.TD_ERR_INVALID_ARG


def test_an_axis_that_would_pass_the_window_limit_is_refused():
    """256 bounded columns 4 apart would gain a 257th window."""
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    engine = _engine()
    g = engine.make_grid(1028, 64, 8, 8, 4, 4)
    assert g.cols == 256
    lo_x, _, lo_y, _ = engine.shift_bounds(g)
    out, before = _sentinel()
    assert _cabi.lib.td_grid_shift(ctypes.byref(g), lo_x, lo_y, 4, ctypes.byref(out)) == _cabi.TD_ERR_UNSUPPORTED
    assert bytes(out) == before
    wrapped = engine.make_grid(1024, 64, 8, 8, 4, 4, wrap=1)   # a periodic axis keeps its 256 windows
    assert wrapped.cols == 256 and engine.shift_grid(wrapped, 3, 1, 4).cols == 256


# ------------------------------------------------------------------------------------------------ the tile method
def _p(w=64, h=48):
    return types.SimpleNamespace(width=w * 8, height=h * 8, sampler_name="Euler a", disable_extra_networks=True)


def _sampler():
    return types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None,
                                                                      step=0), sample_img2img=None)


def _spot(w=64, h=48, tile=(24, 16), overlap=0, bs=4, wrap=0, seed=0):
    from multidiffusion_upscaler_for_automatic1111_b200 import SpotDiffusion
    d = SpotDiffusion(_p(w, h), _sampler())
    d.init_grid_bbox(tile[0], tile[1], overlap, bs, wrap_x=bool(wrap & so.WRAP_X), wrap_y=bool(wrap & so.WRAP_Y), shift_seed=seed)
    return d


def test_method_is_exported():
    import multidiffusion_upscaler_for_automatic1111_b200 as pkg
    from multidiffusion_upscaler_for_automatic1111_b200.tile_methods import SpotDiffusion
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import Method
    assert pkg.SpotDiffusion is SpotDiffusion and "SpotDiffusion" in pkg.__all__
    assert Method("SpotDiffusion") == "SpotDiffusion" and Method.SPOT_DIFF == "SpotDiffusion"


@pytest.mark.parametrize("wrap", WRAPS)
def test_schedule_matches_oracle(wrap):
    d = _spot(wrap=wrap, seed=11)
    b = d._shift_bounds
    assert b == so.bounds(64, 48, 24, 16, 0, wrap)
    assert [d.draw_shift() for _ in range(20)] == so.schedule(11, b, 20)
    again = _spot(wrap=wrap, seed=11)
    other = _spot(wrap=wrap, seed=12)
    seq = [again.draw_shift() for _ in range(20)]
    assert seq == so.schedule(11, b, 20)
    assert [other.draw_shift() for _ in range(20)] != seq


def test_schedule_draws_x_before_y():
    d = _spot(seed=5)
    lo_x, hi_x, lo_y, hi_y = d._shift_bounds
    assert hi_x - lo_x > 1 and hi_y - lo_y > 1
    rng = random.Random(5)
    for _ in range(10):
        sx = rng.randrange(lo_x, hi_x)
        sy = rng.randrange(lo_y, hi_y)
        assert d.draw_shift() == (sx, sy)


def test_single_value_axes_draw_nothing():
    """A 24-wide canvas under a 24-wide tile has one bounded column: only y draws, so the sequence is y's alone."""
    d = _spot(w=24, h=48, seed=3)
    lo_x, hi_x, lo_y, hi_y = d._shift_bounds
    assert (lo_x, hi_x) == (0, 1) and hi_y - lo_y > 1
    rng = random.Random(3)
    assert [d.draw_shift() for _ in range(8)] == [(0, rng.randrange(lo_y, hi_y)) for _ in range(8)]
    both = _spot(w=24, h=16, seed=3)               # one window on both axes: the generator is never touched
    state = both._shift_rng.getstate()
    assert [both.draw_shift() for _ in range(4)] == [(0, 0)] * 4
    assert both._shift_rng.getstate() == state


def test_plan_attributes_describe_the_current_call():
    engine = _engine()
    d = _spot(bs=5)
    g = d._grid
    assert d.num_tiles == g.num_tiles == len([b for bb in d.batched_bboxes for b in bb])
    assert (d.num_batches, d.tile_bs) == (g.num_batches, g.tile_bs)
    base = engine.make_grid(64, 48, 24, 16, 0, 5)
    assert d.num_tiles == (base.cols + 1) * (base.rows + 1)


def test_refused_features_leave_the_delegate_unchanged():
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import BBoxSettings
    d = _spot()
    snapshot = dict(d.__dict__)
    sampler_img2img = d.sampler_raw.sample_img2img
    rows = {0: BBoxSettings(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", "Background", 0.2, -1)}
    with pytest.raises(NotImplementedError):
        d.init_custom_bbox(rows, True, False)
    with pytest.raises(NotImplementedError):
        d.init_tile_shard(None)
    with pytest.raises(NotImplementedError):
        d.init_noise_inverse(10, 1.0, lambda: None, lambda *a: None, 0.5, 64)
    assert d.__dict__.keys() == snapshot.keys()
    assert all(d.__dict__[k] is v for k, v in snapshot.items())
    assert d.sampler_raw.sample_img2img is sampler_img2img
    assert not d.enable_custom_bbox and d.custom_bboxes == [] and not d.noise_inverse_enabled and d._shard is None
