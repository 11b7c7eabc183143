"""Seamless DemoFusion (get_views(..., wrap_x, wrap_y)) on the CPU: the new oracle (tests/demofusion_wrap_oracle.py,
demofusion_views / demofusion_step) against the reference-derived one, the delegate's ring windows and jitter draws, the
new kernel bodies run on the host through tests/emul/, the argument checks of the three new C-ABI entries, and the
delegate on torch stand-ins (unsharded and tile-sharded over gloo)."""
import ctypes
import os
import random
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import demofusion_wrap_oracle as dwo
import wrap_oracle as wo
from conftest import ROOT
from helpers import DTYPES
from oracle import demofusion as odf
from oracle import synth, tiling
from oracle.make_golden import DEMO_CFG, DEMO_JITTER_SEED, demo_denoise, position_aware_denoise

PKG = os.path.join(ROOT, "multidiffusion_upscaler_for_automatic1111_b200")
CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}
WRAPS = {"x": wo.WRAP_X, "y": wo.WRAP_Y, "xy": wo.WRAP_X | wo.WRAP_Y}


def batched(items, bs):
    nb = -(-len(items) // bs)
    tbs = -(-len(items) // nb)
    return [items[i * tbs:(i + 1) * tbs] for i in range(nb)], tbs


def oracle_step(x, windows, mixture, wrap, jr, c=DEMO_CFG, local=None, global_=None):
    """demofusion_wrap_oracle.demofusion_step at DEMO_CFG's scale / cosine settings."""
    N = x.shape[0]
    lb, _ = batched(windows, c["tile_bs"])
    gb, _ = batched(odf.global_views(c["scale"], mixture), c["tile_bs_g"])
    cf = odf.cosine_factor(c["current_step"], c["t_enc"])
    local = local or (lambda t, b: synth.fake_denoise(t, b, N))
    global_ = global_ or (lambda t, b: demo_denoise(t))
    return dwo.demofusion_step(x, lb, gb, c["scale"], mixture, True, c["sig"], cf, c["cs2"], c["cs3"], local, global_, wrap=wrap,
                               jitter_range=jr)


def make_delegate(mixture, jitter, wrap, c=DEMO_CFG, seed=DEMO_JITTER_SEED):
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    p = types.SimpleNamespace(width=c["W"] * 8, height=c["H"] * 8, sampler_name="Euler a", current_scale_num=c["scale"], mixture=mixture,
                              gaussian_filter=True, random_jitter=jitter, cosine_scale_1=c["cs1"], cosine_scale_2=c["cs2"],
                              cosine_scale_3=c["cs3"], current_step=c["current_step"], steps=20, t_enc=c["t_enc"], sd_model=None)
    inner = types.SimpleNamespace(forward=None)
    d = DemoFusion(p, types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=inner, image_cfg_scale=None, forward=None)))
    d.window_size, d.sig = c["window"], c["sig"]
    random.seed(seed)
    d.get_views(c["overlap"], c["tile_bs"], c["tile_bs_g"], wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    return d


def oracle_windows(wrap, jitter, c=DEMO_CFG, seed=DEMO_JITTER_SEED):
    return dwo.demofusion_views(c["W"], c["H"], c["window"], c["overlap"], wrap, random.Random(seed) if jitter else None)


def windows_of(d):
    return [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb]


# ------------------------------------------------------------------------------------------ 1. the oracle at wrap = 0
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("mixture", [True, False], ids=["mixture", "plain"])
@pytest.mark.parametrize("jitter", [False, True], ids=["grid", "jitter"])
def test_oracle_step_without_wrap_equals_the_reference_oracle(dn, mixture, jitter):
    """demofusion_step(wrap = 0) is oracle/demofusion.sample_one_step bit for bit; with jitter the reference oracle gets the
    latent padded by jitter_range and the windows in padded coordinates, and its output is cropped."""
    c, dt = DEMO_CFG, DTYPES[dn]
    x = synth.latent(31, (c["N"], c["C"], c["H"], c["W"]), dt)
    windows, jr = oracle_windows(0, jitter)
    if jitter:
        ref_windows, _, _, ref_jr = tiling.demofusion_views_jitter(c["W"], c["H"], c["window"], c["overlap"], random.Random(DEMO_JITTER_SEED))
        assert jr == ref_jr > 0 and [(a + jr, b + jr, w, h) for a, b, w, h in windows] == ref_windows
    else:
        ref_windows = tiling.demofusion_views(c["W"], c["H"], c["window"], c["overlap"])[0]
        assert jr == 0 and windows == ref_windows
    got = oracle_step(x, windows, mixture, 0, jr)
    lb, _ = batched(ref_windows, c["tile_bs"])
    gb, _ = batched(odf.global_views(c["scale"], mixture), c["tile_bs_g"])
    xp = F.pad(x, (jr, jr, jr, jr), "constant", value=0) if jr else x
    cf = odf.cosine_factor(c["current_step"], c["t_enc"])
    want = odf.sample_one_step(xp, lb, gb, c["scale"], mixture, True, c["sig"], cf, c["cs2"], c["cs3"],
                               lambda t, b: synth.fake_denoise(t, b, c["N"]), lambda t, b: demo_denoise(t), jitter_range=jr)
    if jr:
        want = want[:, :, jr:jr + c["H"], jr:jr + c["W"]]
    assert got.dtype == want.dtype and torch.equal(got, want)
    assert torch.equal(torch.signbit(got), torch.signbit(want))


def test_oracle_blur_is_circular_on_the_wrapped_axes():
    """The blur of a canvas rolled by any amount along a wrapped axis is the rolled blur."""
    x = synth.latent(5, (1, 4, 20, 28), torch.float32)
    for w, dims in ((wo.WRAP_X, (3,)), (wo.WRAP_Y, (2,)), (wo.WRAP_X | wo.WRAP_Y, (2, 3))):
        y = dwo.demofusion_gaussian_filter(x, 7, 0.8, w)
        for d in dims:
            assert torch.allclose(dwo.demofusion_gaussian_filter(torch.roll(x, 5, d), 7, 0.8, w), torch.roll(y, 5, d), rtol=0, atol=1e-6)
    assert torch.equal(dwo.demofusion_gaussian_filter(x, 5, 0.8, 0), odf.gaussian_filter(x, 5, 0.8))


# ------------------------------------------------------------------------------------------ 2. windows and jitter draws
@pytest.mark.parametrize("wn", list(WRAPS))
def test_wrapped_grid_windows_are_the_periodic_plan(wn):
    c, wrap = DEMO_CFG, WRAPS[wn]
    d = make_delegate(False, False, wrap)
    windows, jr = oracle_windows(wrap, False)
    ov = max(0, min(c["overlap"], c["window"] - 4))
    xs = (wo.periodic_origins if wrap & wo.WRAP_X else wo.linear_origins)(c["W"], c["window"], ov)
    ys = (wo.periodic_origins if wrap & wo.WRAP_Y else wo.linear_origins)(c["H"], c["window"], ov)
    assert jr == 0 and windows_of(d) == windows == [(x, y, c["window"], c["window"]) for y in ys for x in xs]
    want = wo.weights(windows, c["W"], c["H"])
    assert want.min() >= 1 and np.array_equal(d._counts.cpu().numpy(), want)


@pytest.mark.parametrize("wn", list(WRAPS))
@pytest.mark.parametrize("seed", [DEMO_JITTER_SEED, 7, 123])
def test_wrapped_jitter_windows_follow_the_seeded_draws(wn, seed):
    """The delegate draws the oracle's windows from Python's `random`; every pixel is covered; origins on a wrapped axis lie
    in [0, L), and on a bounded axis every offset obeys the reference's border rule."""
    c, wrap = DEMO_CFG, WRAPS[wn]
    d = make_delegate(True, True, wrap, seed=seed)
    windows, jr = oracle_windows(wrap, True, seed=seed)
    assert jr == d.jitter_range == 6 and windows_of(d) == windows
    assert list(d._origins_host) == [v for b in windows for v in b[:2]]
    cover = np.zeros((c["H"], c["W"]), np.int32)
    for x, y, w, h in windows:
        iy, oky = dwo.axis_indices(y, h, c["H"], bool(wrap & wo.WRAP_Y))
        ix, okx = dwo.axis_indices(x, w, c["W"], bool(wrap & wo.WRAP_X))
        cover[np.ix_(iy[oky].numpy(), ix[okx].numpy())] += 1
    assert cover.min() >= 1
    base, _ = oracle_windows(wrap, False)
    moved = False
    for (x, y, ws, _), (bx, by, _, _) in zip(windows, base):
        for o, b, L, bit in ((x, bx, c["W"], wo.WRAP_X), (y, by, c["H"], wo.WRAP_Y)):
            if wrap & bit:
                assert 0 <= o < L and (o - b) % L in set(range(0, jr + 1)) | set(range(L - jr, L))
                moved |= o != b
            else:
                at_start, at_end = b == 0, b + ws == L                # demofusion.py:116-134
                lo, hi = (0, 0) if at_start and at_end else (-jr, 0) if at_start else (0, jr) if at_end else (-jr, jr)
                assert lo <= o - b <= hi, (o, b, L)
    assert moved


# ------------------------------------------------------------------------------------------ 3. kernel bodies on the host
def _build_emul(name, harness, deps):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out_dir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, name)
    srcs = [os.path.join(ROOT, "tests", "emul", harness), os.path.join(PKG, "csrc", "td_host.cpp")]
    deps = srcs + [os.path.join(PKG, "csrc", f) for f in deps]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        tmp = so + f".{os.getpid()}.tmp"
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
               "--expt-relaxed-constexpr", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(PKG, "csrc"), "-o", tmp, *srcs]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-3000:]
        os.replace(tmp, so)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def jemul():
    # the same harness as tests/test_jitter_emulation.py, built under its own name
    return _build_emul("libtd_jitter_wrap_emul.so", "jitter_host_emul.cu", ["td_jitter.cu", "td_device.cuh"])


@pytest.fixture(scope="module")
def cemul():
    return _build_emul("libtd_demofusion_emul.so", "demofusion_host_emul.cu", ["td_demofusion.cu", "td_device.cuh"])


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def ring_windows(T, H, W, th, tw, wrap, seed):
    """Windows across the seam on the wrapped axes, hanging off both edges on the bounded ones (negative origins included)."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(T):
        ox = int(rng.integers(0, W)) if wrap & wo.WRAP_X else int(rng.integers(-(tw - 1), W))
        oy = int(rng.integers(0, H)) if wrap & wo.WRAP_Y else int(rng.integers(-(th - 1), H))
        out.append((ox, oy, tw, th))
    if wrap & wo.WRAP_X:
        out[0] = (W - tw // 2, out[0][1], tw, th)                  # straddles the x seam
    else:
        out[0] = (-(tw // 2), out[0][1], tw, th)                   # hangs off the left edge
    if wrap & wo.WRAP_Y:
        out[1] = (out[1][0], H - 1, tw, th)
    else:
        out[1] = (out[1][0], H - th // 3, tw, th)                  # hangs off the bottom edge
    return out


def oracle_list_blend(outs_all, windows, N, shape, dt, wrap):
    """demofusion_step's local blend: x_buffer / max(count, 1), both in dt, from explicit per-window index arrays."""
    H, W = shape[2], shape[3]
    buf, cnt = torch.zeros(shape, dtype=dt), torch.zeros(shape, dtype=dt)
    for t, b in enumerate(windows):
        iy, oky = dwo.axis_indices(b[1], b[3], H, bool(wrap & wo.WRAP_Y))
        ix, okx = dwo.axis_indices(b[0], b[2], W, bool(wrap & wo.WRAP_X))
        idx = (slice(None), slice(None), iy[oky][:, None], ix[okx][None, :])
        buf[idx] = buf[idx] + outs_all[t * N:(t + 1) * N][:, :, oky][:, :, :, okx]
        cnt[idx] = cnt[idx] + 1
    return buf / torch.where(cnt == 0, torch.tensor(1, dtype=dt), cnt)


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wn", ["none", "x", "y", "xy"])
def test_emulated_wrap_list_scatter_and_blend_equal_the_oracle(jemul, dn, wn):
    dt, wrap = DTYPES[dn], WRAPS.get(wn, 0)
    N, C, H, W, th, tw, tile_bs, T = 2, 3, 37, 53, 16, 24, 4, 11
    windows = ring_windows(T, H, W, th, tw, wrap, 3 + wrap)
    flat = np.array([v for b in windows for v in b[:2]], dtype=np.int32)
    x = synth.latent(41, (N, C, H, W), dt)
    x[0, 0, 0, 0] = -0.0
    tiles = torch.empty((T * N, C, th, tw), dtype=dt)
    assert jemul.td_emul_scatter_bboxes_wrap(_p(x), _p(tiles), flat.ctypes.data_as(ctypes.c_void_p), T, N, C, H, W, th, tw, wrap,
                                             x.element_size()) == 0
    want = torch.cat([dwo.demofusion_crop(x, b, wrap) for b in windows], dim=0)
    assert torch.equal(tiles.view(torch.int16 if dt != torch.float32 else torch.int32),
                       want.view(torch.int16 if dt != torch.float32 else torch.int32))

    outs_all = synth.latent(42, (T * N, C, th, tw), dt)
    nb = -(-T // tile_bs)
    outs = [outs_all[b * tile_bs * N:min((b + 1) * tile_bs, T) * N].contiguous() for b in range(nb)]
    ptrs = (ctypes.c_void_p * nb)(*[o.data_ptr() for o in outs])
    got = torch.empty((N, C, H, W), dtype=torch.float32)
    assert jemul.td_emul_blend_bboxes_wrap(ptrs, nb, tile_bs, flat.ctypes.data_as(ctypes.c_void_p), T, N, C, H, W, th, tw, wrap, CODE[dt],
                                           _p(got)) == 0
    want = oracle_list_blend(outs_all, windows, N, (N, C, H, W), dt, wrap)
    assert torch.equal(got.to(dt), want) and torch.equal(torch.signbit(got.to(dt)), torch.signbit(want))


def fmaf_conv_reference(cemul, x, k2, wrap):
    """The stencil's own tap order on an explicitly circularly padded canvas: the bounded body (wrap = 0) on
    F.pad(mode="circular") of the wrapped axes, cropped.  Bit-exact twin of the wrap body when its indexing is right."""
    r = k2.shape[0] // 2
    px, py = (r if wrap & wo.WRAP_X else 0), (r if wrap & wo.WRAP_Y else 0)
    xp = F.pad(x.float(), (px, px, py, py), mode="circular").to(x.dtype).contiguous() if (px or py) else x
    out = torch.empty_like(xp)
    n, c, hh, ww = xp.shape
    assert cemul.td_emul_depthwise_conv2d_wrap(_p(xp), _p(out), n * c, hh, ww, k2.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                               k2.shape[0], 0, CODE[x.dtype]) == 0
    return out[:, :, py:py + x.shape[2], px:px + x.shape[3]]


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wn", ["none", "x", "y", "xy"])
@pytest.mark.parametrize("s", [1, 3, 8])
def test_emulated_wrap_conv_equals_the_oracle(cemul, dn, wn, s):
    dt, wrap = DTYPES[dn], WRAPS.get(wn, 0)
    k = 2 * s - 1
    x = synth.latent(51, (2, 3, 17, 23), dt)
    k2 = odf.gaussian_kernel(k, 0.9, 1)[0, 0].to(dt).float().contiguous().numpy()
    got = torch.empty_like(x)
    assert cemul.td_emul_depthwise_conv2d_wrap(_p(x), _p(got), 6, 17, 23, k2.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), k, wrap,
                                               CODE[dt]) == 0
    assert torch.equal(got, fmaf_conv_reference(cemul, x, k2, wrap))
    want = dwo.demofusion_gaussian_filter(x, k, 0.9, wrap)            # torch's conv: another summation order
    u = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7, torch.float32: 2.0 ** -23}[dt]
    assert (got.float() - want.float()).abs().max().item() <= 2 * u * max(1.0, want.float().abs().max().item())


# ------------------------------------------------------------------------------------------ 4. argument checks
def test_new_entries_refuse_bad_arguments_before_touching_memory():
    """Bogus but non-null device pointers: every call below must be refused by the host checks (a launch would fault)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    lib, bad = _cabi.lib, _cabi.TD_ERR_INVALID_ARG
    fake = ctypes.c_void_p(0x1000)
    k2 = np.full((5, 5), 0.04, np.float32)
    kp = k2.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    conv = lambda H, W, k, wrap, dt=0: lib.td_depthwise_conv2d_wrap(fake, fake, 4, H, W, kp, k, wrap, dt, None)
    assert conv(8, 8, 5, 4) == bad and b"wrap=4" in lib.td_last_error()
    assert conv(8, 8, 5, -1) == bad
    assert conv(8, 1, 5, 1) == bad and b"radius" in lib.td_last_error()        # k/2 = 2 > W = 1 on the wrapped x axis
    assert conv(1, 8, 5, 2) == bad and b"radius" in lib.td_last_error()
    assert conv(8, 8, 4, 3) == bad and conv(8, 8, 17, 3) == bad
    assert conv(8, 8, 5, 3, dt=7) == bad and b"dtype" in lib.td_last_error()
    assert lib.td_depthwise_conv2d_wrap(fake, fake, 4, 8, 8, None, 5, 3, 0, None) == bad

    H, W, th, tw, N, C = 20, 30, 8, 12, 1, 4

    def org(*xy):
        return (ctypes.c_int32 * len(xy))(*xy)
    ptrs = (ctypes.c_void_p * 1)(0x1000)
    out = ctypes.cast(fake, ctypes.POINTER(ctypes.c_float))

    def both(origins, wrap, n=1, tile=(th, tw), dt=0):
        a = lib.td_scatter_bboxes_wrap(fake, fake, fake, origins, n, N, C, H, W, tile[0], tile[1], wrap, dt, None)
        b = lib.td_blend_bboxes_wrap(ptrs, 1, n, fake, origins, n, N, C, H, W, tile[0], tile[1], wrap, dt, out, None)
        return a, b
    assert both(org(0, 0), 4) == (bad, bad)
    assert both(None, 1) == (bad, bad) and b"missing" in lib.td_last_error()
    assert both(None, 0) == (bad, bad)
    assert both(org(W, 0), 1) == (bad, bad) and b"out of range" in lib.td_last_error()     # wrapped x: 0 <= o < W
    assert both(org(-1, 0), 1) == (bad, bad)
    assert both(org(0, H), 2) == (bad, bad) and both(org(0, -1), 2) == (bad, bad)
    assert both(org(-tw, 0), 2) == (bad, bad)                                            # bounded x: o >= -(tw-1)
    assert both(org(W, 0), 2) == (bad, bad)                                              # bounded x: o <= W-1
    assert both(org(0, -th), 1) == (bad, bad) and both(org(0, H), 1) == (bad, bad)
    assert both(org(0, 0), 1, tile=(th, W + 1)) == (bad, bad) and b"exceeds" in lib.td_last_error()
    assert both(org(0, 0), 2, tile=(H + 1, tw)) == (bad, bad)
    assert both(org(0, 0, 3, 3), 3, n=2, dt=9) == (bad, bad)
    assert lib.td_blend_bboxes_wrap(ptrs, 1, 2, fake, org(0, 0, -tw, 0), 2, N, C, H, W, th, tw, 2, 0, out, None) == bad
    assert lib.td_blend_bboxes_wrap(ptrs, 1, 1, None, org(0, 0), 1, N, C, H, W, th, tw, 1, 0, out, None) == bad


# ------------------------------------------------------------------------------------------ 5. the delegate on stand-ins
def install_wrap_stand_ins(set_attr=setattr):
    """helpers.install_demofusion_stand_ins plus wrap-aware torch stand-ins for the entries a seamless canvas reaches."""
    from helpers import install_demofusion_stand_ins
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion, engine
    install_demofusion_stand_ins(set_attr)

    def bbs(g):
        return [tuple(int(v) for v in r) for r in engine.grid_bboxes_xywh(g)]

    def scatter_tiles(g, x, out=None, tile_begin=0, tile_end=None, flags=0):
        return torch.cat([dwo.demofusion_crop(x, b, int(g.wrap)) for b in bbs(g)[tile_begin:tile_end]], dim=0)

    def blend_multidiffusion(g, outs, N, C, tile_bs, weights, acc_dtype, x_buffer=None, flags=0, out=None, rcp_weights=None):
        allt = torch.cat(list(outs), dim=0)
        return oracle_list_blend(allt, bbs(g), N, (N, C, g.H, g.W), acc_dtype, int(g.wrap)).float()

    def scatter_bboxes(x, origins_dev, origins_host, n_tiles, tile_h, tile_w, out=None, wrap=0):
        return torch.cat([dwo.demofusion_crop(x, (ox, oy, tile_w, tile_h), wrap) for ox, oy in origins_dev.view(-1, 2).tolist()], dim=0)

    def blend_bboxes(batch_outs, tile_bs, origins_dev, origins_host, n_tiles, N, C, H, W, tile_h, tile_w, wrap=0):
        allt = torch.cat(list(batch_outs), dim=0)
        windows = [(ox, oy, tile_w, tile_h) for ox, oy in origins_dev.view(-1, 2).tolist()]
        return oracle_list_blend(allt, windows, N, (N, C, H, W), allt.dtype, wrap).float()

    for name, fn in dict(scatter_tiles=scatter_tiles, blend_multidiffusion=blend_multidiffusion, scatter_bboxes=scatter_bboxes,
                         blend_bboxes=blend_bboxes).items():
        set_attr(engine, name, fn)
    set_attr(DemoFusion, "gaussian_filter", lambda self, latents, kernel_size=3, sigma=1.0:
             dwo.demofusion_gaussian_filter(latents, kernel_size, sigma, self._wrap))


CASES = [(j, dn, m, wn) for j in (False, True) for dn, m in (("f32", True), ("f32", False), ("f16", True)) for wn in WRAPS]


def _run_delegate(jitter, dn, mixture, wrap, shard=False):
    c = DEMO_CFG
    dt = DTYPES[dn]
    x = synth.latent(31, (c["N"], c["C"], c["H"], c["W"]), dt)
    d = make_delegate(mixture, jitter, wrap)
    d.sampler_forward = position_aware_denoise(d)
    windows, jr = oracle_windows(wrap, jitter)
    assert windows_of(d) == windows
    want = oracle_step(x, windows, mixture, wrap, jr)
    if shard:
        d.init_tile_shard(None)
    d.cosine_factor = odf.cosine_factor(c["current_step"], c["t_enc"])
    cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8)], "c_concat": [torch.zeros(c["N"], 5, 1, 1)]}
    got = d.sample_one_step(x, torch.ones(c["N"]), cond)
    assert got.dtype == dt and got.shape == want.shape == x.shape
    tol = 3e-6 if dn == "f32" else 2e-3
    err = (got.float() - want.float()).abs().max().item()
    assert err <= tol * max(1.0, want.float().abs().max().item()), f"jitter={jitter} {dn} mixture={mixture} wrap={wrap}: max err {err}"
    return got


@pytest.mark.parametrize("jitter,dn,mixture,wn", CASES, ids=[f"{'jitter' if j else 'grid'}-{dn}-{'mix' if m else 'plain'}-{wn}"
                                                             for j, dn, m, wn in CASES])
def test_delegate_on_cpu_stand_ins_equals_the_oracle(monkeypatch, jitter, dn, mixture, wn):
    install_wrap_stand_ins(monkeypatch.setattr)
    _run_delegate(jitter, dn, mixture, WRAPS[wn])


def test_delegate_crops_a_canvas_sized_icond_through_the_ring_windows(monkeypatch):
    """mode 0 (local windows) crops a canvas-sized c_concat with the latent's modular / zero-fill rule; mode 1 is unchanged."""
    install_wrap_stand_ins(monkeypatch.setattr)
    c = DEMO_CFG
    for wrap in WRAPS.values():
        d = make_delegate(False, True, wrap)
        icond = synth.latent(9, (c["N"], 5, c["H"], c["W"]), torch.float32)
        cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8)], "c_concat": [icond]}
        bbs = d.batched_bboxes[0]
        got = d.repeat_cond_dict(cond, bbs, 0)["c_concat"][0]
        assert torch.equal(got, torch.cat([dwo.demofusion_crop(icond, (b.x, b.y, b.w, b.h), wrap) for b in bbs], dim=0))
        views = d.global_batched_bboxes[0]
        s = c["scale"]
        got = d.repeat_cond_dict(cond, views, 1)["c_concat"][0]
        assert torch.equal(got, torch.cat([icond[:, :, by::s, bx::s] for bx, by in views], dim=0))


def test_forward_one_step_and_get_noise_do_not_pad_a_seamless_canvas(monkeypatch):
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    c = DEMO_CFG
    monkeypatch.setattr(DemoFusion, "is_kdiff", property(lambda self: True))
    for wrap in WRAPS.values():
        d = make_delegate(True, True, wrap)
        seen = []
        d.sample_one_step = lambda x_in, sigma, cond: (seen.append(tuple(x_in.shape)), x_in * 2)[1]
        d.t_enc = c["t_enc"]
        x = synth.latent(3, (c["N"], c["C"], c["H"], c["W"]), torch.float32)
        d.p.x, d.p.noise = x, x
        out = d.get_noise(x, torch.ones(c["N"]), {"c_crossattn": [torch.zeros(c["N"], 77, 8)]}, 0)
        assert out.shape == x.shape and seen[-1] == tuple(x.shape) and torch.equal(out, x * 2)
        cfg = d.sampler.model_wrap_cfg
        cfg.forward_ori = lambda x_in, sigma, **kw: cfg.inner_model.forward(x_in, sigma, None)
        d.sampler_forward = None
        out = d.forward_one_step(x, torch.ones(c["N"]))
        assert out.shape == x.shape and seen[-1] == tuple(x.shape)


# ------------------------------------------------------------------------------------------ 5b. tile shard over gloo
def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_worker(rank, world, port, result_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        install_wrap_stand_ins()
        for jitter, dn, mixture, wn in [(False, "f32", True, "xy"), (True, "f32", True, "x"), (True, "f16", False, "xy"), (False, "f16", False, "y")]:
            single = _run_delegate(jitter, dn, mixture, WRAPS[wn])
            sharded = _run_delegate(jitter, dn, mixture, WRAPS[wn], shard=True)
            assert torch.equal(sharded, single), f"rank {rank}: sharded {jitter} {dn} {wn} differs from the unsharded delegate"
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_sharded_wrapped_delegate_equals_unsharded(tmp_path, world):
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
