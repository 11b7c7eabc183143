"""Inpainting on the GPU: td_grid_active_tiles against the numpy restatement of the rule (tests/test_inpaint_mask_plan.py),
the sparse blends against the dense ones (bit patterns, every dtype, random / empty / full active sets, more than
TD_MAX_BATCH_PTRS compact batches, the form that ran, the slot-table refusals), and the MultiDiffusion / Mixture of Diffusers
delegates end to end: a masked sampler loop with init_inpaint_mask against the same loop without it."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal
from test_gpu_blend_limits import K_ASYNC, K_GENERIC, K_MOD_ASYNC, forms, launched, template_args
from test_inpaint_mask_plan import JUST_BELOW_ONE, rule

pytestmark = pytest.mark.gpu


def _engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


def _bbs(g):
    return [tuple(int(v) for v in r) for r in _engine().grid_bboxes_xywh(g)]


# Which kernel ran is read from a CUPTI trace, which is reliable only in a young process (late in a long GPU session profiler
# sessions come back without kernel records, see tests/test_gpu_wrap_forms.py).  So the form assertions run in a fresh
# interpreter (`test_launched_forms_in_a_fresh_process`); in this process `_traced` only runs the call, and every bit check
# runs in both.
FORMS_CHILD = os.environ.get("TD_INPAINT_FORMS_CHILD") == "1"
FORM_TESTS = "sparse_blend_against_dense or more_than_128"


def _traced(fn):
    """The kernel names `fn` launched (in the child interpreter), or None after running it (elsewhere)."""
    if not FORMS_CHILD:
        fn()
        return None
    return launched(fn)


def test_launched_forms_in_a_fresh_process():
    """The sparse-blend tests rerun in a fresh interpreter, where they also assert which kernel form ran."""
    if FORMS_CHILD:
        pytest.skip("already the child interpreter")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    cmd = [sys.executable, *flags, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k", FORM_TESTS]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(cmd, cwd=root, env=dict(os.environ, TD_INPAINT_FORMS_CHILD="1"), capture_output=True, text=True, timeout=1200)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail


CFG2 = (512, 512, 96, 96, 48, 8)
BIG = (1024, 1024, 96, 96, 48, 8)


# ------------------------------------------------------------------------------------------------ td_grid_active_tiles
def _masks(W, H, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    out = {"ones": torch.ones((H, W)), "zeros": torch.zeros((H, W))}
    m = torch.ones((H, W))
    idx = torch.randint(0, H * W, (6,), generator=g)
    m.view(-1)[idx] = torch.rand(6, generator=g)
    out["sparse"] = m
    for name, val in (("nan", float("nan")), ("below_one", JUST_BELOW_ONE), ("corner", 0.0)):
        m = torch.ones((H, W))
        m[H - 1, W - 1] = val if name == "corner" else m[H - 1, W - 1]
        if name != "corner":
            m[H // 2, 47] = val                        # a tile edge of the 96 / 48 plans
        out[name] = m
    blob = torch.ones((4, H, W))
    blob[3, H // 3:H // 3 + 40, W // 2:W // 2 + 40] = 0.25
    out["chw_last_plane"] = blob
    out["nchw"] = blob.unsqueeze(0).repeat(2, 1, 1, 1)
    return {k: v.to(dtype) for k, v in out.items()}


@pytest.mark.parametrize("geom", [CFG2, BIG], ids=["cfg2", "1024"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_active_tiles_match_rule(geom, dn):
    engine = _engine()
    W, H, tw, th, ov, bs = geom
    g = engine.make_grid(W, H, tw, th, ov, bs)
    for name, m in _masks(W, H, DTYPES[dn], 3).items():
        got = engine.active_tiles(g, m.cuda())
        want = rule(m, _bbs(g))
        assert np.array_equal(got, want), f"{dn} {name}: {np.flatnonzero(got != want)}"
    m = torch.ones((H, W), dtype=DTYPES[dn])
    m[192:320, 192:320] = 0
    n = int(engine.active_tiles(g, m.cuda()).sum())
    print(f"{W}x{H}: a 128^2 latent square in the middle reaches {n} of {g.num_tiles} tiles")


def test_active_tiles_refusals_leave_output_untouched():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    engine = _engine()
    g = engine.make_grid(256, 192, 96, 96, 48, 4)
    m = torch.zeros((4, 192, 256), dtype=torch.float16, device="cuda")
    out = torch.full((g.num_tiles + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    stream = _cabi.current_stream_ptr()
    wrapped = engine.make_grid(256, 192, 96, 96, 48, 4, wrap=engine.WRAP_X)
    leaves = _cabi.TdGrid.from_buffer_copy(g)
    leaves.xs[leaves.cols - 1] = g.W - g.tile_w + 1

    def call(grid=g, mask=m.data_ptr(), planes=4, dtype=_cabi.TD_F16, dst=out.data_ptr()):
        return _cabi.lib.td_grid_active_tiles(ctypes.byref(grid) if grid is not None else None, mask, planes, dtype, dst, stream)
    cases = [dict(mask=None), dict(mask=m.data_ptr() + 1), dict(dst=None), dict(planes=0), dict(planes=-1), dict(dtype=7),
             dict(grid=None), dict(grid=leaves)]
    for kw in cases:
        assert call(**kw) == _cabi.TD_ERR_INVALID_ARG, (kw, _cabi.lib.td_last_error())
    assert call(grid=wrapped) == _cabi.TD_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (out == 0xA5).all()
    assert call() == _cabi.TD_OK
    torch.cuda.synchronize()
    assert (out[:g.num_tiles] == 1).all() and (out[g.num_tiles:] == 0xA5).all()
    with pytest.raises(ValueError):
        engine.active_tiles(g, m[:, :, :128])


# ------------------------------------------------------------------------------------------------ sparse blends
def _tile_outputs(g, N, C, dt, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn((g.num_tiles * N, C, g.tile_h, g.tile_w), generator=gen) * 2).to(dt).cuda()


def _batches(t, n_tiles, N, tile_bs):
    return [t[i * N:min(i + tile_bs, n_tiles) * N] for i in range(0, n_tiles, tile_bs)]


def _coverage(g, active):
    total = torch.zeros((g.H, g.W), dtype=torch.int32)
    kept = torch.zeros((g.H, g.W), dtype=torch.int32)
    for t, (x, y, w, h) in enumerate(_bbs(g)):
        total[y:y + h, x:x + w] += 1
        kept[y:y + h, x:x + w] += int(active[t])
    return total, kept


def _run_pair(method, g, N, C, dt, acc_dt, active, flags=0, seed=0):
    """(sparse, dense with the skipped tiles' outputs zeroed, dense), each (x_out or None, x_buffer); and the form names."""
    engine = _engine()
    tiles = _tile_outputs(g, N, C, dt, seed)
    idx = torch.tensor([t for t in range(g.num_tiles) if active[t]], dtype=torch.long)
    rows = (idx[:, None] * N + torch.arange(N)[None, :]).reshape(-1).cuda()
    compact = tiles.index_select(0, rows)
    zeroed = tiles.clone().view(g.num_tiles, N, C, g.tile_h, g.tile_w)
    zeroed[torch.from_numpy(~active).cuda()] = 0
    zeroed = zeroed.view_as(tiles)
    slot = engine.slot_table(active)
    slot_dev = torch.from_numpy(slot).cuda()
    bs = g.tile_bs
    res = {}
    if method == "md":
        w = torch.from_numpy(engine.grid_weights(g)).cuda()
        for key, src, n in (("dense", tiles, g.num_tiles), ("zeroed", zeroed, g.num_tiles)):
            xb = torch.empty((N, C, g.H, g.W), dtype=acc_dt, device="cuda")
            xo = engine.blend_multidiffusion(g, _batches(src, n, N, bs), N, C, bs, w, acc_dt, x_buffer=xb, flags=flags)
            res[key] = (xo, xb)
        xb = torch.full((N, C, g.H, g.W), float("nan"), dtype=acc_dt, device="cuda")
        box = {}
        names = _traced(lambda: box.setdefault("xo", engine.blend_multidiffusion_sparse(
            g, _batches(compact, len(idx), N, bs), N, C, bs, w, acc_dt, slot_dev, slot, x_buffer=xb, flags=flags, tile_dtype=dt)))
        res["sparse"] = (box["xo"], xb)
    else:
        tw_ = torch.from_numpy(_engine_gauss(g)).cuda()
        rf = torch.from_numpy(engine.rescale_factor(engine.grid_weights(g, _engine_gauss(g)))).cuda()
        for key, src, n in (("dense", tiles, g.num_tiles), ("zeroed", zeroed, g.num_tiles)):
            xb = torch.empty((N, C, g.H, g.W), dtype=acc_dt, device="cuda")
            engine.blend_mixture(g, _batches(src, n, N, bs), N, C, bs, tw_, rf, xb, flags=flags)
            res[key] = (None, xb)
        xb = torch.full((N, C, g.H, g.W), float("nan"), dtype=acc_dt, device="cuda")
        names = _traced(lambda: engine.blend_mixture_sparse(g, _batches(compact, len(idx), N, bs), N, C, bs, tw_, rf, xb, slot_dev, slot,
                                                             flags=flags, tile_dtype=dt))
        res["sparse"] = (None, xb)
    torch.cuda.synchronize()
    return res, names


def _engine_gauss(g):
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import gaussian_weights
    return gaussian_weights(g.tile_w, g.tile_h).cpu().numpy()


def _check(method, g, res, active, what):
    total, kept = _coverage(g, active)
    full = (kept == total).view(1, 1, g.H, g.W)
    none = (kept == 0).view(1, 1, g.H, g.W)
    for i in (0, 1):
        got, dense, zeroed = res["sparse"][i], res["dense"][i], res["zeroed"][i]
        if got is None:
            continue
        got, dense, zeroed = got.cpu(), dense.cpu(), zeroed.cpu()
        sel = full.expand_as(got)
        assert_bit_equal(got[sel], dense[sel], f"{what}: pixels all of whose tiles are active")
        z = none.expand_as(got)
        assert_bit_equal(got[z], torch.zeros_like(got[z]), f"{what}: pixels no active tile covers")
        # partly covered pixels: the dense blend with the skipped tiles' outputs zeroed.  MultiDiffusion's accumulator is never -0, so
        # adding +0 changes nothing; Mixture of Diffusers' can be -0, and -0 + (+0) = +0 where the sparse blend keeps -0
        assert_bit_equal(got, zeroed, f"{what}: against zeroed skipped tiles", allow_signed_zero=(method == "mod"))


def _active_sets(T, seed):
    rng = np.random.default_rng(seed)
    return {"random": rng.random(T) < 0.4, "empty": np.zeros(T, bool), "full": np.ones(T, bool)}


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_sparse_blend_against_dense_cp_async(method, dn):
    engine = _engine()
    g = engine.make_grid(256, 192, 64, 64, 24, 4)
    dt = DTYPES[dn]
    for name, active in _active_sets(g.num_tiles, 5).items():
        res, names = _run_pair(method, g, 2, 4, dt, dt, active)
        if names is not None:
            kernel = K_ASYNC if method == "md" else K_MOD_ASYNC
            assert forms(names) == {kernel}, sorted(names)
            assert [a[-1] for a in template_args(names, kernel)] == ["true"], sorted(names)
        _check(method, g, res, active, f"{method} {dn} {name}")


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("case", ["force_generic", "mixed_dtypes", "odd_width"])
def test_sparse_blend_against_dense_generic(method, case):
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    engine = _engine()
    W = 250 if case == "odd_width" else 256
    g = engine.make_grid(W, 136, 64, 64, 24, 3)
    dt, acc = (torch.float32, torch.float16) if case == "mixed_dtypes" else (torch.bfloat16, torch.bfloat16)
    flags = _cabi.TD_FLAG_FORCE_GENERIC if case == "force_generic" else 0
    for name, active in _active_sets(g.num_tiles, 6).items():
        res, names = _run_pair(method, g, 1, 4, dt, acc, active, flags=flags)
        if names is not None:
            assert forms(names) == {K_GENERIC}, sorted(names)
            assert [a[-1] for a in template_args(names, K_GENERIC)] == ["true"], sorted(names)
        _check(method, g, res, active, f"{method} {case} {name}")


@pytest.mark.parametrize("method", ["md", "mod"])
def test_sparse_blend_more_than_128_compact_batches(method):
    """tile_bs 1 and about 300 active tiles: the compact batches are concatenated to fit TD_MAX_BATCH_PTRS, as the dense blends'."""
    engine = _engine()
    g = engine.make_grid(512, 512, 32, 32, 8, 1)
    active = np.random.default_rng(8).random(g.num_tiles) < 0.7
    assert g.num_tiles > 400 and active.sum() > 128
    res, names = _run_pair(method, g, 1, 4, torch.float16, torch.float16, active)
    if names is not None:
        assert forms(names) == {K_ASYNC if method == "md" else K_MOD_ASYNC}, sorted(names)
        assert any("cat" in n.lower() for n in names if not forms([n])), sorted(names)
    _check(method, g, res, active, f"{method} >128 batches")


@pytest.mark.parametrize("method", ["md", "mod"])
def test_bad_slot_tables_are_refused(method):
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    engine = _engine()
    g = engine.make_grid(256, 192, 64, 64, 24, 4)
    N, C, T = 1, 4, g.num_tiles
    active = np.zeros(T, bool)
    active[[0, 3, 5]] = True
    tiles = _tile_outputs(g, N, C, torch.float16, 1)[:3 * N]
    good = engine.slot_table(active)
    w = torch.from_numpy(engine.grid_weights(g)).cuda()
    tw_ = torch.from_numpy(_engine_gauss(g)).cuda()
    out = torch.full((N, C, g.H, g.W), 7.0, device="cuda")
    xb = torch.full((N, C, g.H, g.W), 7.0, dtype=torch.float16, device="cuda")
    ptrs = (ctypes.c_void_p * 1)(tiles.data_ptr())
    stream = _cabi.current_stream_ptr()

    def call(slot, n=T, dev=None, nb=1, flags=0, grid=g):
        host = np.ascontiguousarray(slot, dtype=np.int32)
        d = torch.from_numpy(np.resize(host, max(n, T))).cuda() if dev is None else dev
        hp = host.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        dp = d if isinstance(d, int) or d is None else d.data_ptr()
        if method == "md":
            return _cabi.lib.td_blend_multidiffusion_sparse(ctypes.byref(grid), ptrs, nb, 4, N, C, _cabi.TD_F16, _cabi.TD_F16, w.data_ptr(),
                                                            None, out.data_ptr(), xb.data_ptr(), dp, hp, n, flags, stream)
        return _cabi.lib.td_blend_mixture_sparse(ctypes.byref(grid), ptrs, nb, 4, N, C, _cabi.TD_F16, _cabi.TD_F16, tw_.data_ptr(),
                                                 w.data_ptr(), xb.data_ptr(), dp, hp, n, flags, stream)
    out_of_range = good.copy(); out_of_range[5] = 3
    duplicate = good.copy(); duplicate[5] = 1
    below = good.copy(); below[7] = -2
    gap = good.copy(); gap[5] = -1; gap[3] = 2             # positions {0, 2}: 1 unused, 2 out of range for K = 2
    wrapped = engine.make_grid(256, 192, 64, 64, 24, 4, wrap=engine.WRAP_X)
    for kw in (dict(slot=out_of_range), dict(slot=duplicate), dict(slot=below), dict(slot=gap), dict(slot=good[:-1], n=T - 1),
               dict(slot=np.append(good, -1), n=T + 1), dict(slot=good, dev=0), dict(slot=good, dev=torch.from_numpy(good).cuda().data_ptr() + 2),
               dict(slot=good, nb=2), dict(slot=good, flags=_cabi.TD_FLAG_TMA), dict(slot=good, flags=_cabi.TD_FLAG_ROWS)):
        assert call(**kw) == _cabi.TD_ERR_INVALID_ARG, (kw, _cabi.lib.td_last_error())
    wrapped_slots = np.full(wrapped.num_tiles, -1, dtype=np.int32)
    wrapped_slots[[0, 3, 5]] = [0, 1, 2]
    assert call(wrapped_slots, n=wrapped.num_tiles, grid=wrapped) == _cabi.TD_ERR_UNSUPPORTED, _cabi.lib.td_last_error()
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (xb == 7.0).all()
    assert call(good) == _cabi.TD_OK
    torch.cuda.synchronize()
    assert not (xb == 7.0).all()


# ------------------------------------------------------------------------------------------------ delegates end to end
W, H, N, C = 160, 128, 2, 4
TILE, OV, BS = 48, 16, 3


def _unet(x_tile, t, cond):
    """Per-sample deterministic stand-in for the UNet (a sample's output depends on that sample only): the zero-padded tile blur
    plus the window's crop of the spatial image cond, plus a fraction of the hint / StableSR crops the UNet sees."""
    icond = cond["c_concat"][0] if isinstance(cond, dict) else None
    out = wo.blur_denoise(x_tile).float()
    if icond is not None and tuple(icond.shape[2:]) == tuple(x_tile.shape[2:]):
        out = out + icond.float()
    return out.to(x_tile.dtype)


@pytest.fixture
def shared():
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
    model = types.SimpleNamespace(cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="concat"))
    host.use_shared(types.SimpleNamespace(state=state, sd_model=model))
    host._a1111_cache.clear()
    yield model
    host.use_shared(None)


def _sampler(kdiff, forward):
    cls = type("KDiffusionSampler" if kdiff else "CompVisSampler", (), {})
    s = cls()
    s.model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=forward), image_cfg_scale=None, step=0)
    return s


def _rows(kind):
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import BlendMode
    bg, fg = BlendMode.BACKGROUND.value, BlendMode.FOREGROUND.value
    if kind is None:
        return None
    rows = {0: (True, 0.0, 0.0, 0.3, 0.3, "kept corner", "", bg, 0.2, -1),      # inside the kept area: skipped
            1: (True, 0.35, 0.3, 0.3, 0.4, "masked middle", "", bg, 0.2, -1)}
    if kind == "fg":
        rows[2] = (True, 0.7, 0.65, 0.3, 0.35, "kept fg", "", fg, 0.3, 5)
        rows[3] = (True, 0.4, 0.35, 0.3, 0.3, "masked fg", "", fg, 0.5, 3)
    return rows


def _delegate(method, kdiff, calls, regions, side, shared, mask=None):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion

    def unet(x, t, cond=None, *a, **k):
        calls.append(("tile", x.shape[0], side["unit"].hint_cond.cpu() if side else None,
                      side["sr"].latent_image.cpu() if side and side["sr"].latent_image is not None else None))
        return _unet(x, t, cond)
    p = types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True)
    if method == "md":
        d = MultiDiffusion(p, _sampler(kdiff, unet))
        region_fn = lambda x, *a, **k: (calls.append(("region", x.shape[0], None, None)), _unet(x, None, None))[1]
        d.kdiff_custom_forward = region_fn
        d.ddim_custom_forward = region_fn
    else:
        shared.__dict__.pop("apply_model_original_md", None)      # hook() keeps an earlier delegate's original otherwise
        shared.apply_model = lambda x, t, cond: unet(x, t, cond)
        d = MixtureOfDiffusers(p, _sampler(kdiff, None))
        d.custom_apply_model = lambda x, *a, **k: (calls.append(("region", x.shape[0], None, None)), _unet(x, None, None))[1]
    d.init_grid_bbox(TILE, TILE, OV, BS)
    if regions is not None:
        d.init_custom_bbox(regions, True, False)
    if mask is not None:
        d.init_inpaint_mask(mask)
    if side:
        d.init_controlnet(types.SimpleNamespace(latest_network=types.SimpleNamespace(control_params=[side["unit"]])), False)
        d.init_stablesr(types.SimpleNamespace(stablesr_model=side["sr"]))
        side["sr"].set_image_hooks["TiledDiffusion"](side["sr_latent"].cuda())
    d.init_done()
    d.hook()
    return d


def _model_call(d, method, x, t, cond):
    if method == "md":
        return d.sampler.model_wrap_cfg.inner_model.forward(x, t, cond=cond)
    return d._sd_model().apply_model(x, t, cond)


def _sample(d, method, kdiff, init, mask, cond, steps=4):
    """The WebUI's masked loops with a stub denoiser: k-diffusion Euler with `denoised = init * mask + nmask * denoised`, or a
    DDIM-style loop that masks x before every call; the final latent is composited with init as img2img does."""
    nmask = 1 - mask
    x = init + torch.randn(init.shape, generator=torch.Generator().manual_seed(9)).to(init.dtype).cuda()
    sigmas = [1.0, 0.6, 0.3, 0.1, 0.0][:steps + 1]
    for i in range(steps):
        if kdiff:
            den = _model_call(d, method, x, torch.full((N,), sigmas[i], device="cuda"), cond)
            den = init * mask + nmask * den
            x = (x + (x - den) / sigmas[i] * (sigmas[i + 1] - sigmas[i])).to(init.dtype)
        else:
            x = init * mask + nmask * x
            out = _model_call(d, method, x, torch.full((N,), float(10 * i), device="cuda"), cond)
            x = (x * 0.75 + out * 0.25).to(init.dtype)
    return x * nmask + init * mask


def _mask(dt):
    m = torch.ones((1, 1, H, W), dtype=dt)
    m[:, :, 50:80, 60:100] = 0.0
    m[:, :, 48:50, 58:102] = 0.5                     # a soft edge
    return m.cuda()


@pytest.mark.parametrize("side_inputs", [False, True], ids=["plain", "controlnet_stablesr"])
@pytest.mark.parametrize("regions", [None, "bg", "fg"])
@pytest.mark.parametrize("kdiff", [True, False], ids=["euler", "ddim"])
@pytest.mark.parametrize("method", ["md", "mod"])
def test_masked_sampling_matches_full_plan(shared, method, kdiff, regions, side_inputs):
    dt = torch.float16
    gen = torch.Generator().manual_seed(4)
    init = torch.randn((N, C, H, W), generator=gen).to(dt).cuda()
    icond = torch.randn((N, C, H, W), generator=gen).to(dt).cuda()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4, device="cuda")], "c_concat": [icond]}
    mask = _mask(dt)
    results, runs = {}, {}
    for use_mask in (False, True):
        side = None
        if side_inputs:
            side = dict(unit=types.SimpleNamespace(hint_cond=torch.randn((1, 3, H * 8, W * 8), generator=torch.Generator().manual_seed(5)).half().cuda()),
                        sr=types.SimpleNamespace(set_image_hooks={}, latent_image=None),
                        sr_latent=torch.randn((1, 4, H, W), generator=torch.Generator().manual_seed(6)).half())
        calls = []
        d = _delegate(method, kdiff, calls, _rows(regions), side, shared, mask=mask if use_mask else None)
        results[use_mask] = _sample(d, method, kdiff, init, mask, cond).cpu()
        runs[use_mask] = (d, calls)
    full, masked = results[False], results[True]
    m = mask.cpu().expand_as(full)
    assert_bit_equal(masked[m < 1], full[m < 1], "pixels with mask < 1")
    assert_bit_equal(masked[m == 1], init.cpu()[m == 1], "kept pixels")
    d, calls = runs[True]
    ip = d._inpaint
    tile_calls = [c for c in calls if c[0] == "tile"]
    assert 0 < len(ip.batched_bboxes) < d.num_batches
    assert len(tile_calls) == 4 * len(ip.batched_bboxes), "one UNet call per active batch and step"
    n_regions = sum(1 for c in calls if c[0] == "region")
    assert n_regions == 4 * sum(ip.regions) and (regions is None or not all(ip.regions))
    if side_inputs:
        # the hint / StableSR crops the UNet receives for an active tile are the full run's crops of that tile
        fd, fcalls = runs[False]
        full_tile = {}
        for (kind, n, hint, sr), bboxes in zip([c for c in fcalls if c[0] == "tile"], fd.batched_bboxes * 4):
            for j, b in enumerate(bboxes):
                full_tile[(b.x, b.y)] = (_rows_of(hint, j, len(bboxes), kdiff), sr[j:j + 1] if sr is not None else None)
        for (kind, n, hint, sr), bboxes in zip(tile_calls, ip.batched_bboxes * 4):
            for j, b in enumerate(bboxes):
                want_hint, want_sr = full_tile[(b.x, b.y)]
                assert_bit_equal(_rows_of(hint, j, len(bboxes), kdiff), want_hint, "hint crop of an active tile")
                assert_bit_equal(sr[j:j + 1], want_sr, "StableSR crop of an active tile")


def _rows_of(hint, j, n_tiles, kdiff):
    """Tile j's rows of the hint batch a UNet call receives (k-diffusion: each tile's N copies adjacent; DDIM: the batch repeated)."""
    return hint[j * N:(j + 1) * N] if kdiff else hint[j:j + 1]


@pytest.mark.parametrize("method", ["md", "mod"])
def test_keep_everything_returns_zeros_without_unet_calls(shared, method):
    calls = []
    d = _delegate(method, True, calls, None, None, shared, mask=torch.ones((H, W), device="cuda"))
    x = torch.randn((N, C, H, W)).half().cuda()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4, device="cuda")], "c_concat": [x]}
    out = _model_call(d, method, x, torch.ones(N, device="cuda"), cond)
    torch.cuda.synchronize()
    assert calls == [] and d.total_bboxes == 0
    assert out.dtype == (torch.float32 if method == "md" else torch.float16)
    assert_bit_equal(out.cpu(), torch.zeros(out.shape, dtype=out.dtype), "the blend of nothing")


@pytest.mark.parametrize("method", ["md", "mod"])
def test_noise_inversion_runs_the_full_plan(shared, method):
    """get_noise has no host mask: the inverted latent is the same with and without init_inpaint_mask, bit for bit."""
    dt = torch.float32
    gen = torch.Generator().manual_seed(12)
    x0 = torch.randn((1, C, H, W), generator=gen).to(dt).cuda()
    cond = {"c_crossattn": [torch.zeros(1, 2, 4, device="cuda")], "c_concat": [torch.randn((1, C, H, W), generator=gen).cuda()]}
    out = {}
    for use_mask in (False, True):
        if method == "md":
            shared.apply_model = lambda x, t, cond: _unet(x, t, cond)
        d = _delegate(method, True, [], None, None, shared, mask=_mask(dt) if use_mask else None)
        x = x0
        for k in range(3):
            x = x + d.get_noise(x, torch.full((1,), 0.5 + k), cond, 3 - k).float() * 0.1
        out[use_mask] = x.cpu()
        assert d._inpaint is None or not d._full_plan_pass
    assert_bit_equal(out[True], out[False], "inverted latent")
