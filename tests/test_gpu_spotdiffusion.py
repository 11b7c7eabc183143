"""SpotDiffusion on the GPU: td_grid_counts bit for bit against td_grid_weights + td_rescale_factor, its refusals, and the tile
method's consecutive denoiser calls against tests/spot_oracle.py on the k-diffusion and DDIM paths, with the ControlNet and
StableSR crops of each call's plan."""
import ctypes
import types

import numpy as np
import pytest
import torch

import spot_oracle as so
import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal

pytestmark = pytest.mark.gpu

WRAPS = [0, so.WRAP_X, so.WRAP_X | so.WRAP_Y]


def _engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


def _host_counts(g):
    engine = _engine()
    w = engine.grid_weights(g)
    with np.errstate(divide="ignore"):
        return w.reshape(-1), engine.rescale_factor(w).reshape(-1)


def _device_counts(g, rcp=True):
    n = g.H * g.W
    w = torch.full((n,), float("nan"), device="cuda")
    r = torch.full((n,), float("nan"), device="cuda")
    _engine().grid_counts(g, w, r if rcp else None)
    torch.cuda.synchronize()
    return w.cpu(), r.cpu()


@pytest.mark.parametrize("wrap", [0, so.WRAP_X, so.WRAP_Y, so.WRAP_X | so.WRAP_Y])
@pytest.mark.parametrize("overlap", [0, 8, 48])
@pytest.mark.parametrize("tile", [64, 96, 128])
@pytest.mark.parametrize("L", [64, 97, 150, 513])
def test_counts_bit_equal_to_host_weights(L, tile, overlap, wrap):
    engine = _engine()
    h = {64: 150, 97: 64, 150: 97, 513: 512}[L]
    g = engine.make_grid(L, h, tile, tile, overlap, 4, wrap=wrap)
    lo_x, hi_x, lo_y, hi_y = engine.shift_bounds(g)
    for sx, sy in {(lo_x, lo_y), (hi_x - 1, hi_y - 1), ((lo_x + hi_x) // 2, (lo_y + hi_y) // 2)}:
        s = engine.shift_grid(g, sx, sy, 4)
        want_w, want_r = _host_counts(s)
        got_w, got_r = _device_counts(s)
        assert_bit_equal(got_w, torch.from_numpy(want_w), f"weights {L} {tile} {overlap} {wrap} ({sx}, {sy})")
        assert_bit_equal(got_r, torch.from_numpy(want_r), "reciprocals")
        got_w, untouched = _device_counts(s, rcp=False)
        assert_bit_equal(got_w, torch.from_numpy(want_w), "weights without reciprocals")
        assert torch.isnan(untouched).all()


def _hand_plan(W, H, tw, th, xs, ys, wrap=0):
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
    g = TdGrid()
    g.W, g.H, g.tile_w, g.tile_h, g.wrap = W, H, tw, th, wrap
    g.cols, g.rows = len(xs), len(ys)
    g.num_tiles = g.num_batches = g.cols * g.rows
    g.tile_bs = 1
    for i, v in enumerate(xs):
        g.xs[i] = v
    for i, v in enumerate(ys):
        g.ys[i] = v
    return g


@pytest.mark.parametrize("W", [1, 2, 3, 5, 7, 97, 1031])
def test_counts_on_one_row_and_odd_widths(W):
    """W not a multiple of the 4-float vector, one-row canvases (the tail stores), and a one-column one."""
    engine = _engine()
    plans = [engine.make_grid(W, 1, 64, 64, 8, 4), engine.make_grid(W, 1, 64, 64, 8, 4, wrap=3), engine.make_grid(W, 3, 8, 2, 0, 4)]
    plans.append(engine.shift_grid(plans[0], *engine.shift_bounds(plans[0])[::2], 4))
    plans.append(_hand_plan(1, W, 1, max(1, W // 2), [0], sorted({0, W // 3, W - max(1, W // 2)})))
    plans.append(_hand_plan(W, 2, W, 2, sorted({0, W // 2}), [0, 1], wrap=3))        # tiles as wide as the canvas, off 0
    for g in plans:
        want_w, want_r = _host_counts(g)
        got_w, got_r = _device_counts(g)
        assert_bit_equal(got_w, torch.from_numpy(want_w), f"W={W} {g.W}x{g.H}")
        assert_bit_equal(got_r, torch.from_numpy(want_r), f"W={W} reciprocals")


def test_counts_refusals_leave_the_outputs_untouched():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
    engine = _engine()
    good = engine.shift_grid(engine.make_grid(150, 97, 64, 64, 8, 4), 1, 1, 4)
    n = good.W * good.H
    buf = torch.full((n + 8,), float("nan"), device="cuda")
    rbuf = torch.full((n + 8,), float("nan"), device="cuda")
    stream = _cabi.current_stream_ptr()

    def call(g, w=None, r=None):
        w = buf.data_ptr() if w is None else w
        r = rbuf.data_ptr() if r is None else r
        return _cabi.lib.td_grid_counts(ctypes.byref(g) if g is not None else None, w, r, stream)

    leaves = TdGrid.from_buffer_copy(good)
    leaves.xs[leaves.cols - 1] = good.W - good.tile_w + 1
    decreasing = TdGrid.from_buffer_copy(good)
    decreasing.ys[1], decreasing.ys[2] = good.ys[2], good.ys[1]
    wrapped_out = TdGrid.from_buffer_copy(good)
    wrapped_out.wrap = 1
    wrapped_out.xs[0] = good.W                             # a periodic origin must lie in [0, W)
    empty = TdGrid.from_buffer_copy(good)
    empty.rows = 0
    huge = _hand_plan(32768, 1, 8, 1, [0], [0])
    cases = [(leaves, {}, _cabi.TD_ERR_INVALID_ARG), (decreasing, {}, _cabi.TD_ERR_INVALID_ARG), (wrapped_out, {}, _cabi.TD_ERR_INVALID_ARG),
             (empty, {}, _cabi.TD_ERR_INVALID_ARG), (None, {}, _cabi.TD_ERR_INVALID_ARG), (good, {"w": 0}, _cabi.TD_ERR_INVALID_ARG),
             (good, {"w": buf.data_ptr() + 4}, _cabi.TD_ERR_INVALID_ARG), (good, {"r": rbuf.data_ptr() + 8}, _cabi.TD_ERR_INVALID_ARG),
             (huge, {}, _cabi.TD_ERR_UNSUPPORTED)]
    for g, kw, want in cases:
        assert call(g, **kw) == want, (kw, _cabi.lib.td_last_error())
    torch.cuda.synchronize()
    assert torch.isnan(buf).all() and torch.isnan(rbuf).all()
    assert call(good) == _cabi.TD_OK                       # and the same buffers take a valid plan
    torch.cuda.synchronize()
    assert not torch.isnan(buf[:n]).any() and torch.isnan(buf[n:]).all()


# ------------------------------------------------------------------------------------------------ the tile method
W, H, N, C = 64, 48, 2, 4
TW, TH = 24, 16
CALLS = 5


def _p():
    return types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True)


def _sampler(kdiff, forward):
    cls = type("KDiffusionSampler" if kdiff else "CompVisSampler", (), {})
    s = cls()
    s.model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=forward), image_cfg_scale=None, step=0)
    return s


def _unet(x_tile, t, cond):
    """Position-dependent stand-in for the UNet: a zero-padded tile blur (depends on where a pixel sits in its window) plus the
    window's crop of the spatial image cond (depends on where the window sits on the canvas).  IEEE adds only: CPU and GPU
    agree bit for bit."""
    icond = cond["c_concat"][0]
    return (wo.blur_denoise(x_tile).float() + icond.float()).to(x_tile.dtype)


def _oracle_unet(icond):
    def denoise(x_tile, bboxes):
        return (wo.blur_denoise(x_tile).float() + wo.scatter(icond, bboxes).float()).to(x_tile.dtype)
    return denoise


@pytest.fixture
def shared():
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
    model = types.SimpleNamespace(cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="concat"))
    host.use_shared(types.SimpleNamespace(state=state, sd_model=model))
    host._a1111_cache.clear()
    yield state
    host.use_shared(None)


def _spot(kdiff, wrap, overlap, bs, seed=0, forward=_unet):
    from multidiffusion_upscaler_for_automatic1111_b200 import SpotDiffusion
    d = SpotDiffusion(_p(), _sampler(kdiff, forward))
    assert d.is_kdiff == kdiff
    d.init_grid_bbox(TW, TH, overlap, bs, wrap_x=bool(wrap & so.WRAP_X), wrap_y=bool(wrap & so.WRAP_Y), shift_seed=seed)
    d.init_done()
    d.hook()
    return d


def _inputs(dtype, seed):
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn((N, C, H, W), generator=gen) * 2).to(dtype)
    icond = torch.randn((N, C, H, W), generator=gen).to(dtype)
    cond = {"c_crossattn": [torch.zeros(N, 2, 4).cuda()], "c_concat": [icond.cuda()]}
    return x, icond, cond


def _call(d, x, cond):
    return d.sampler.model_wrap_cfg.inner_model.forward(x.cuda(), torch.ones(N).cuda(), cond=cond)


@pytest.mark.parametrize("kdiff", [True, False], ids=["kdiff", "ddim"])
@pytest.mark.parametrize("bs", [1, 4, 1000], ids=["bs1", "bs4", "bsall"])
@pytest.mark.parametrize("overlap", [0, 8])
@pytest.mark.parametrize("wrap", WRAPS, ids=["bounded", "wrapx", "wrapxy"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_consecutive_calls_match_oracle(shared, dn, wrap, overlap, bs, kdiff):
    d = _spot(kdiff, wrap, overlap, bs, seed=7)
    x, icond, cond = _inputs(DTYPES[dn], 1)
    shifts = so.schedule(7, so.bounds(W, H, TW, TH, overlap, wrap), CALLS)
    denoise = _oracle_unet(icond)
    seen = set()
    for k, (sx, sy) in enumerate(shifts):
        got = _call(d, x, cond)
        plan = so.SpotPlan(W, H, TW, TH, overlap, bs, wrap, sx, sy)
        assert [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb] == plan.bboxes, f"call {k}"
        assert (d.num_tiles, d.num_batches, d.tile_bs) == (len(plan.bboxes), plan.num_batches, plan.tile_bs)
        assert_bit_equal(got.cpu(), so.step(x, plan, denoise), f"{dn} wrap={wrap} ov={overlap} bs={bs} kdiff={kdiff} call {k}")
        assert_bit_equal(d.weights.view(H, W).cpu(), torch.from_numpy(plan.weights), "count canvas")
        seen.add((sx, sy))
        x = got.cpu().to(x.dtype)
    assert len(seen) > 1, "the windows never moved"


def test_same_seed_same_results(shared):
    x, _, cond = _inputs(torch.float16, 2)
    a, b = _spot(True, so.WRAP_X, 0, 4, seed=3), _spot(True, so.WRAP_X, 0, 4, seed=3)
    c = _spot(True, so.WRAP_X, 0, 4, seed=4)
    xa = xb = xc = x
    differs = False
    for _ in range(CALLS):
        ra, rb, rc = _call(a, xa, cond), _call(b, xb, cond), _call(c, xc, cond)
        assert torch.equal(ra, rb)
        differs |= not torch.equal(ra, rc)
        xa, xb, xc = ra.half().cpu(), rb.half().cpu(), rc.half().cpu()
    assert differs


@pytest.mark.parametrize("kdiff", [True, False], ids=["kdiff", "ddim"])
@pytest.mark.parametrize("wrap", [0, so.WRAP_X | so.WRAP_Y], ids=["bounded", "wrapxy"])
def test_side_inputs_are_cropped_with_each_calls_plan(shared, kdiff, wrap):
    """ControlNet hints (x8) and the StableSR latent seen per batch are the crops of that call's plan, not of the first one."""
    hint = torch.randn((1, 3, H * 8, W * 8), generator=torch.Generator().manual_seed(5)).half()
    sr_latent = torch.randn((1, 4, H, W), generator=torch.Generator().manual_seed(6)).half()
    unit = types.SimpleNamespace(hint_cond=hint.cuda())
    sr_model = types.SimpleNamespace(set_image_hooks={}, latent_image=None)
    seen = []

    def forward(x_tile, t, cond):
        seen.append((unit.hint_cond.cpu(), sr_model.latent_image.cpu()))
        return _unet(x_tile, t, cond)
    d = _spot(kdiff, wrap, 0, 4, seed=9, forward=forward)
    d.init_controlnet(types.SimpleNamespace(latest_network=types.SimpleNamespace(control_params=[unit])), False)
    d.init_stablesr(types.SimpleNamespace(stablesr_model=sr_model))
    sr_model.set_image_hooks["TiledDiffusion"](sr_latent.cuda())
    x, icond, cond = _inputs(torch.float16, 3)
    for k, (sx, sy) in enumerate(so.schedule(9, so.bounds(W, H, TW, TH, 0, wrap), 3)):
        seen.clear()
        got = _call(d, x, cond)
        plan = so.SpotPlan(W, H, TW, TH, 0, 4, wrap, sx, sy)
        assert_bit_equal(got.cpu(), so.step(x, plan, _oracle_unet(icond)), f"call {k}")
        assert len(seen) == plan.num_batches
        for bbs, (crops, sr) in zip(plan.batched_bboxes, seen):
            want = wo.scatter(hint, [(bx * 8, by * 8, bw * 8, bh * 8) for (bx, by, bw, bh) in bbs])
            want = want.repeat_interleave(N, dim=0) if kdiff else want.repeat([N * 2, 1, 1, 1])
            assert_bit_equal(crops, want, f"hint crop, call {k}")
            assert_bit_equal(sr, wo.scatter(sr_latent, bbs), f"StableSR crop, call {k}")
        x = got.cpu().half()


def test_hires_pass_and_interrupt(shared):
    """Another latent size goes to the model untiled and draws no shift; an interrupt returns the input, like MultiDiffusion."""
    d = _spot(True, 0, 0, 4, seed=1)
    state = d._shift_rng.getstate()
    big = torch.randn((N, C, H * 2, W * 2)).cuda()
    assert d.sample_one_step(big, lambda t: t * 2, None, None).equal(big * 2)
    assert d._shift_rng.getstate() == state
    x, _, cond = _inputs(torch.float16, 4)
    shared.interrupted = True
    xd = x.cuda()
    assert d.sampler.model_wrap_cfg.inner_model.forward(xd, torch.ones(N).cuda(), cond=cond) is xd
