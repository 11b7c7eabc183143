"""DemoFusion's local-window path (the window-list kernels of csrc/td_jitter.cu behind engine.scatter_bboxes /
engine.blend_bboxes, and the count-normalised grid blend) at the window counts the UI reaches: window 16-256, overlap up
to window - 4 (stride 4), window batches of 1-8, latents up to 1024^2.

Every check compares with a plain reference built from per-window loops, run eagerly in torch on the device:
  scatter  == slicing + torch.cat (bounded), explicit modular index arrays (wrap)                          bit for bit
  blend    == oracle/demofusion.local_blend / demofusion_wrap_oracle.local_blend: the buffer accumulated window by
              window in the latent dtype, divided by the exact fp32 count, in fp32                          bit for bit
  step     == oracle.demofusion.sample_one_step / demofusion_wrap_oracle.demofusion_step at coverage 1024,
              with the tolerances of test_gpu_demofusion_kernels.py::test_sample_one_step_matches_oracle

Jittered window lists of more than 128 batches reach the C entries folded to at most 128 tensors (the spy on `lib` asserts
the table that arrived).  The coverage test puts 4096 windows over one pixel, past the 256 (bf16) and 2048 (fp16) where a
count kept in the latent dtype stops growing, in a tile batch of more than 2^31 elements; it prints its wall times and its
peak device memory (run pytest with -s to see them).

The file name sorts it after test_gpu_vae_kernels.py, for the reason given at the top of test_gpu_zz_sparse_spot_forms.py:
it adds minutes to the pytest process.
"""
import ctypes
import random
import time

import numpy as np
import pytest
import torch

import demofusion_wrap_oracle as dwo
import wrap_oracle as wo
from helpers import DTYPES
from oracle import demofusion as odf
from oracle import synth, tiling
from oracle.make_golden import demo_denoise
from test_demofusion_wrap import ring_windows
from test_gpu_demofusion_kernels import CS2, CS3, SEED, SIG, _delegate

pytestmark = pytest.mark.gpu

WRAP_XY = wo.WRAP_X | wo.WRAP_Y
MAX_PTRS = 128                       # TD_MAX_BATCH_PTRS
LIST_ENTRIES = ("td_blend_bboxes", "td_blend_bboxes_wrap")


def _eng():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


@pytest.fixture
def blend_calls(monkeypatch):
    """(entry, num_batches, tile_bs, batch pointers) of every list-blend call that reaches the C entries."""
    eng = _eng()
    real, calls = eng.lib, []

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name not in LIST_ENTRIES:
                return fn

            def record(ptrs, nb, tile_bs, *rest):
                calls.append((name, nb, tile_bs, [ptrs[i] for i in range(nb)]))
                return fn(ptrs, nb, tile_bs, *rest)
            return record
    monkeypatch.setattr(eng, "lib", Spy())
    return calls


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _origins(windows):
    flat = [int(v) for b in windows for v in b[:2]]
    return torch.tensor(flat, dtype=torch.int32, device="cuda"), (ctypes.c_int32 * len(flat))(*flat)


def _crop(x, b, wrap):
    if wrap:
        return dwo.demofusion_crop(x, b, wrap)
    return x[:, :, b[1]:b[1] + b[3], b[0]:b[0] + b[2]]


def check_scatter(tiles, x, windows, wrap, N, group=64):
    for i in range(0, len(windows), group):
        want = torch.cat([_crop(x, b, wrap) for b in windows[i:i + group]], dim=0)
        assert torch.equal(_bits(tiles[i * N:i * N + want.shape[0]]), _bits(want)), f"windows {i}..{i + group - 1}"


def batches_of(outs_all, T, N, tile_bs):
    return [outs_all[b * tile_bs * N:min((b + 1) * tile_bs, T) * N] for b in range(-(-T // tile_bs))]


def window_outs(outs_all, T, N):
    return [outs_all[t * N:(t + 1) * N] for t in range(T)]


def ref_blend(x_like, windows, outs, wrap):
    return dwo.local_blend(x_like, windows, outs, wrap) if wrap else odf.local_blend(x_like, windows, outs)


def assert_table(calls, wrap, nb, tile_bs, T, batches):
    """One call reached the C entry, with the batch table folded as engine._fit_batch_table does."""
    assert len(calls) == 1, calls
    name, n, bs, ptrs = calls.pop()
    assert name == LIST_ENTRIES[bool(wrap)]
    k = -(-nb // MAX_PTRS)
    assert n == -(-nb // k) <= MAX_PTRS and bs == tile_bs * k
    assert (n - 1) * bs < T <= n * bs
    if k == 1:                                  # no copy below the limit: the caller's own tensors
        assert ptrs == [b.data_ptr() for b in batches]


def run_list(calls, x, windows, tile_bs, wrap, N, origins=None, outs_all=None):
    """Scatter x through the window list, blend the tile outputs (per-window power-of-two scales of the tiles unless
    given) through engine.blend_bboxes, and check both against the references and the table that reached the C entry."""
    eng = _eng()
    T, th, tw = len(windows), windows[0][3], windows[0][2]
    C, H, W = x.shape[1], x.shape[2], x.shape[3]
    od, oh = origins if origins is not None else _origins(windows)
    tiles = eng.scatter_bboxes(x, od, oh, T, th, tw, wrap=wrap)
    assert tiles.shape == (T * N, C, th, tw)
    check_scatter(tiles, x, windows, wrap, N)
    if outs_all is None:
        outs_all = synth.fake_denoise(tiles, windows, N)
    batches = batches_of(outs_all, T, N, tile_bs)
    got = eng.blend_bboxes(batches, tile_bs, od, oh, T, N, C, H, W, th, tw, wrap=wrap)
    assert_table(calls, wrap, len(batches), tile_bs, T, batches)
    want = ref_blend(x, windows, window_outs(outs_all, T, N), wrap)
    assert torch.equal(_bits(got), _bits(want))
    return got, want


# ------------------------------------------------------------------------------------------------ 1. pointer-table boundary
TABLE = [(nb, bs) for nb in (127, 128, 129, 257) for bs in (1, 3, 8)]


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("nb,tile_bs", TABLE, ids=[f"nb{nb}-bs{bs}" for nb, bs in TABLE])
def test_batch_table_at_the_pointer_limit(blend_calls, nb, tile_bs, dn):
    """127 .. 257 window batches, the last one partial when tile_bs > 1, on the bounded and the wrap-xy entry; a 12 x 16
    window on a 40 x 56 canvas."""
    dt = DTYPES[dn]
    N, C, H, W, th, tw = 2, 4, 40, 56, 12, 16
    T = (nb - 1) * tile_bs + max(1, tile_bs - 1)
    rng = np.random.default_rng(10 * nb + tile_bs)
    x = synth.latent(nb + tile_bs, (N, C, H, W), dt).cuda()
    outs_all = synth.latent(7 * nb + tile_bs, (T * N, C, th, tw), dt).cuda()
    for wrap in (0, WRAP_XY):
        if wrap:
            windows = ring_windows(T, H, W, th, tw, wrap, nb + tile_bs)
        else:
            windows = [(int(rng.integers(0, W - tw + 1)), int(rng.integers(0, H - th + 1)), tw, th) for _ in range(T)]
        run_list(blend_calls, x, windows, tile_bs, wrap, N, outs_all=outs_all)


# ------------------------------------------------------------------------------------------------ 2. the UI's window lists
def ui_delegate(L, window, overlap, tile_bs, wrap=0):
    """The delegate's own get_views on an L x L latent, seeded: split_bboxes_jitter (bounded) or split_bboxes_jitter_wrap."""
    d = _delegate(1, False, True, L, L, 1)
    d.window_size = window
    random.seed(SEED)
    d.get_views(overlap, tile_bs, 1, wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    return d


def windows_of(d):
    return [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb]


UI_LISTS = [(512, 128, 96, 1, 169, 169), (1024, 64, 32, 4, 961, 241), (256, 128, 124, 8, 1089, 137)]


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("L,window,overlap,tile_bs,T,nb", UI_LISTS, ids=[f"{c[0]}-w{c[1]}-o{c[2]}-bs{c[3]}" for c in UI_LISTS])
def test_ui_jitter_window_lists(blend_calls, L, window, overlap, tile_bs, T, nb, dn):
    """Random-jitter windows from the delegate's split_bboxes_jitter under a fixed seed, on the latent padded by the jitter
    range, through the delegate's own origin arrays and batch size."""
    d = ui_delegate(L, window, overlap, tile_bs)
    assert (d.num_tiles, d.num_batches) == (T, nb) and d.jitter_range > 0
    windows = windows_of(d)
    Lp = L + 2 * d.jitter_range
    assert min(min(b[0], b[1]) for b in windows) >= 0 and max(max(b[0], b[1]) for b in windows) + window <= Lp
    x = synth.latent(L + window, (2, 4, Lp, Lp), DTYPES[dn]).cuda()
    run_list(blend_calls, x, windows, d.tile_bs, 0, 2, origins=(d._origins_dev.cuda(), d._origins_host))


WRAP_LISTS = {"x": wo.WRAP_X, "y": wo.WRAP_Y, "xy": WRAP_XY}


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wn", list(WRAP_LISTS))
def test_ui_wrap_jitter_window_lists(blend_calls, wn, dn):
    """split_bboxes_jitter_wrap on a 256^2 latent, window 64 / overlap 48, batch size 1: 208 (x, y) or 256 (xy) batches.
    Two more windows sit at the bounded axis' extremes -(tile - 1) and L - 1 (or across both seams at wrap xy)."""
    wrap, L, ws = WRAP_LISTS[wn], 256, 64
    d = ui_delegate(L, ws, 48, 1, wrap)
    windows = windows_of(d)
    assert len(windows) == (256 if wrap == WRAP_XY else 208)
    if wrap == wo.WRAP_X:
        windows += [(5, -(ws - 1), ws, ws), (L - 3, L - 1, ws, ws)]
    elif wrap == wo.WRAP_Y:
        windows += [(-(ws - 1), 7, ws, ws), (L - 1, L - 2, ws, ws)]
    else:
        windows += [(L - 1, L - 1, ws, ws), (L - ws // 2, 0, ws, ws)]
    x = synth.latent(31 + wrap, (2, 4, L, L), DTYPES[dn]).cuda()
    run_list(blend_calls, x, windows, 1, wrap, 2)


# ------------------------------------------------------------------------------------------------ 3. coverage 4096, > 2^31 elements
@pytest.mark.parametrize("dn", list(DTYPES))
def test_coverage_4096_in_a_tile_batch_past_2_31_elements(blend_calls, dn, record_property):
    """512^2, window 256 / overlap 252 (stride 4), N = 2, C = 4, batch size 8: 4225 windows in 529 batches (folded to 106
    tensors of 40), 4096 of them over the canvas centre, 2.2e9 tile elements.  The tile outputs are the scattered tiles
    scaled in place by a power of two per window (exact), so the test holds one tile batch plus the folded copy."""
    eng, dt = _eng(), DTYPES[dn]
    N, C, L, ws, ov, tile_bs = 2, 4, 512, 256, 252, 8
    windows, _, stride = tiling.demofusion_views(L, L, ws, ov)
    T = len(windows)
    assert T == 4225 and stride == 4 and T * N * C * ws * ws > 2 ** 31
    cov = eng.axis_coverage(sorted({b[0] for b in windows}), L, ws, False)
    assert int(cov.max()) ** 2 == 4096
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    x = synth.latent(4225, (N, C, L, L), dt).cuda()
    od, oh = _origins(windows)

    t0 = time.perf_counter()
    tiles = eng.scatter_bboxes(x, od, oh, T, ws, ws)
    torch.cuda.synchronize()
    t_scatter = time.perf_counter() - t0
    check_scatter(tiles, x, windows, 0, N, group=65)
    scales = torch.tensor([synth.tile_scale(b[0], b[1]) for b in windows], dtype=torch.float32, device="cuda").to(dt)
    tiles.view(T, -1).mul_(scales[:, None])
    batches = batches_of(tiles, T, N, tile_bs)

    t0 = time.perf_counter()
    got = eng.blend_bboxes(batches, tile_bs, od, oh, T, N, C, L, L, ws, ws)
    torch.cuda.synchronize()
    t_blend = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    assert_table(blend_calls, 0, len(batches), tile_bs, T, batches)
    want = odf.local_blend(x, windows, window_outs(tiles, T, N))
    assert torch.equal(_bits(got), _bits(want))

    tile_bytes = tiles.numel() * tiles.element_size()
    line = (f"coverage 4096 {dn}: scatter {t_scatter:.3f} s, blend (fold + kernel) {t_blend:.3f} s, peak {peak / 2 ** 30:.2f} GiB "
            f"(tile batch {tile_bytes / 2 ** 30:.2f} GiB) on {torch.cuda.get_device_name()}")
    print(line)
    record_property("coverage_4096", line)
    assert peak < 2.2 * tile_bytes


# ------------------------------------------------------------------------------------------------ 4. edges
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("wrap", [0, WRAP_XY], ids=["bounded", "wrap_xy"])
def test_edges(blend_calls, wrap, N, dn):
    """A window equal to the whole canvas; non-square windows (9 x 14) in the four corners, the last at (W - tw, H - th),
    and one overlapping the first, leaving pixels no window covers (exactly +0 there); a NaN plane and +-inf planes in
    two windows' outputs, which reach exactly the pixels those windows cover."""
    dt = DTYPES[dn]
    C, H, W = 4, 37, 53
    x = synth.latent(N + 3 * wrap, (N, C, H, W), dt).cuda()

    whole = [(0, 0, W, H)] * 3
    run_list(blend_calls, x, whole, 2, wrap, N)

    th, tw = 9, 14
    windows = [(0, 0, tw, th), (W - tw, 0, tw, th), (0, H - th, tw, th), (8, 5, tw, th), (W - tw, H - th, tw, th)]
    outs_all = synth.latent(77 + N, (len(windows) * N, C, th, tw), dt).cuda()
    got, want = run_list(blend_calls, x, windows, 2, wrap, N, outs_all=outs_all)
    count = torch.zeros((H, W), device="cuda")
    for b in windows:
        count[b[1]:b[1] + b[3], b[0]:b[0] + b[2]] += 1
    assert (count == 0).any() and (count > 1).any()
    assert torch.equal(_bits(got[:, :, count == 0]), torch.zeros_like(_bits(got[:, :, count == 0])))

    specials = outs_all.clone()
    specials[3 * N:4 * N, 0] = float("nan")            # window 3, plane c = 0
    specials[4 * N:5 * N, 1] = float("inf")            # window 4 (the last corner), c = 1 and 2
    specials[4 * N:5 * N, 2] = -float("inf")
    got = _eng().blend_bboxes(batches_of(specials, 5, N, 2), 2, *_origins(windows), 5, N, C, H, W, th, tw, wrap=wrap)
    blend_calls.clear()
    want = ref_blend(x, windows, window_outs(specials, 5, N), wrap)
    foot = lambda b: torch.zeros((H, W), dtype=torch.bool, device="cuda").index_fill_(0, torch.arange(b[1], b[1] + th, device="cuda"), True) \
        & torch.zeros((H, W), dtype=torch.bool, device="cuda").index_fill_(1, torch.arange(b[0], b[0] + tw, device="cuda"), True)
    nan_at = torch.zeros_like(got, dtype=torch.bool)
    nan_at[:, 0] = foot(windows[3])
    assert torch.equal(torch.isnan(got), nan_at) and torch.equal(torch.isnan(want), nan_at)
    assert torch.equal(got[:, 1] == float("inf"), foot(windows[4]).expand(N, H, W))
    assert torch.equal(got[:, 2] == -float("inf"), foot(windows[4]).expand(N, H, W))
    assert torch.equal(_bits(got[~nan_at]), _bits(want[~nan_at]))


# ------------------------------------------------------------------------------------------------ 5. whole step at coverage 1024
STEP_MODES = {"jitter": (True, 0), "grid": (False, 0), "wrap_xy_jitter": (True, WRAP_XY)}


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("mixture", [False, True], ids=["plain", "mixture"])
@pytest.mark.parametrize("mode", list(STEP_MODES))
def test_sample_one_step_at_coverage_1024(mode, mixture, dn):
    """DemoFusion.sample_one_step at 256^2, window 128 / overlap 124, batch size 4, scale 2 (the grid and random jitter:
    1089 windows in 273 batches; seamless xy with jitter: 4096 ring windows in 1024 batches) against the fixed oracles."""
    jitter, wrap = STEP_MODES[mode]
    dt, L, ws, ov, s, N, C = DTYPES[dn], 256, 128, 124, 2, 2, 4
    d = _delegate(s, mixture, jitter, L, L, 3)
    d.window_size = ws
    random.seed(SEED)
    d.get_views(ov, 4, 3, wrap_x=bool(wrap), wrap_y=bool(wrap))
    if wrap:
        local, jr = dwo.demofusion_views(L, L, ws, ov, wrap, random.Random(SEED))
        assert (d.num_tiles, d.num_batches) == (4096, 1024)
    elif jitter:
        local, _, _, jr = tiling.demofusion_views_jitter(L, L, ws, ov, random.Random(SEED))
        assert (d.num_tiles, d.num_batches) == (1089, 273)
    else:
        (local, _, _), jr = tiling.demofusion_views(L, L, ws, ov), 0
        assert (d.num_tiles, d.num_batches) == (1089, 273)
    assert windows_of(d) == local and d.jitter_range == jr
    x = synth.latent(2024 + s, (N, C, L, L), dt)
    lb = [local[i * d.tile_bs:(i + 1) * d.tile_bs] for i in range(d.num_batches)]
    views = odf.global_views(s, mixture)
    gb = [views[i * d.global_tile_bs:(i + 1) * d.global_tile_bs] for i in range(d.global_num_batches)]
    local_fn, global_fn = (lambda t, b: synth.fake_denoise(t, b, N)), (lambda t, b: demo_denoise(t))
    if wrap:
        xin = x
        want = dwo.demofusion_step(x, lb, gb, s, mixture, True, SIG, d.cosine_factor, CS2, CS3, local_fn, global_fn, wrap=wrap,
                                   jitter_range=jr)
    else:
        xin = torch.nn.functional.pad(x, (jr, jr, jr, jr), "constant", value=0) if jr else x
        want = odf.sample_one_step(xin, lb, gb, s, mixture, True, SIG, d.cosine_factor, CS2, CS3, local_fn, global_fn, jitter_range=jr)
    cond = {"c_crossattn": [torch.zeros(N, 77, 8, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
    got = d.sample_one_step(xin.cuda(), torch.ones(N, device="cuda"), cond)
    assert got.dtype == dt and got.shape == want.shape
    tol = {torch.float32: 3e-6, torch.float16: 2e-3, torch.bfloat16: 1.6e-2}[dt]
    err = (got.cpu().float() - want.float()).abs().max().item()
    assert err <= tol * max(1.0, want.float().abs().max().item()), f"{mode}: max err {err}"


# ------------------------------------------------------------------------------------------------ 6. refusals
def _refusal_args():
    """A valid engine.blend_bboxes call: 7 windows of 12 x 16 on a 40 x 56 canvas in batches of 3 (3, 3, 1), N = 2, C = 4."""
    N, C, H, W, th, tw, T, bs = 2, 4, 40, 56, 12, 16, 7, 3
    windows = [(3 * t, 2 * t, tw, th) for t in range(T)]
    outs_all = synth.latent(5, (T * N, C, th, tw), torch.float16).cuda()
    od, oh = _origins(windows)
    return dict(batch_outs=batches_of(outs_all, T, N, bs), tile_bs=bs, origins_dev=od, origins_host=oh, n_tiles=T, N=N, C=C, H=H,
                W=W, tile_h=th, tile_w=tw)


def _replace(lst, i, t):
    lst = list(lst)
    lst[i] = t
    return lst


REFUSALS = {
    "one_batch_short": lambda a: dict(batch_outs=a["batch_outs"][:-1]),
    "one_batch_extra": lambda a: dict(batch_outs=a["batch_outs"] + a["batch_outs"][-1:]),
    "tile_bs_mismatch": lambda a: dict(tile_bs=2),
    "tile_bs_0": lambda a: dict(tile_bs=0),
    "partial_batch_full_size": lambda a: dict(batch_outs=_replace(a["batch_outs"], 2, a["batch_outs"][0])),
    "window_transposed": lambda a: dict(batch_outs=[t.transpose(2, 3) for t in a["batch_outs"]]),
    "channels": lambda a: dict(batch_outs=[t[:, :3] for t in a["batch_outs"]]),
    "mixed_dtypes": lambda a: dict(batch_outs=_replace(a["batch_outs"], 1, a["batch_outs"][1].float())),
    "mixed_devices": lambda a: dict(batch_outs=_replace(a["batch_outs"], 1, a["batch_outs"][1].cpu())),
    "cpu_batches": lambda a: dict(batch_outs=[t.cpu() for t in a["batch_outs"]]),
    "origins_int64": lambda a: dict(origins_dev=a["origins_dev"].long()),
    "origins_short": lambda a: dict(origins_dev=a["origins_dev"][:-2]),
    "origins_long": lambda a: dict(origins_dev=torch.cat([a["origins_dev"], a["origins_dev"][:2]])),
    "origins_strided": lambda a: dict(origins_dev=a["origins_dev"].repeat_interleave(2)[::2]),
    "origins_on_cpu": lambda a: dict(origins_dev=a["origins_dev"].cpu()),
    "origins_host_short": lambda a: dict(origins_host=(ctypes.c_int32 * 12)(*a["origins_host"][:12])),
    "origins_host_missing": lambda a: dict(origins_host=None),
}


@pytest.mark.parametrize("wrap", [0, WRAP_XY], ids=["bounded", "wrap_xy"])
@pytest.mark.parametrize("case", list(REFUSALS))
def test_blend_bboxes_refuses_bad_tables_before_any_launch(blend_calls, case, wrap):
    """Each bad argument raises ValueError and no C entry is reached: the tile outputs and the origins are left as they
    were.  The unchanged arguments blend, and a non-contiguous batch is made contiguous and blends the same."""
    a = _refusal_args()
    bad = REFUSALS[case](a)
    if case == "origins_strided":
        assert not bad["origins_dev"].is_contiguous() and torch.equal(bad["origins_dev"], a["origins_dev"])
    sentinels = [t.clone() for t in a["batch_outs"]] + [a["origins_dev"].clone()]
    with pytest.raises(ValueError):
        _eng().blend_bboxes(**{**a, **bad}, wrap=wrap)
    assert blend_calls == []
    for t, s in zip(a["batch_outs"] + [a["origins_dev"]], sentinels):
        assert torch.equal(_bits(t) if t.is_floating_point() else t, _bits(s) if s.is_floating_point() else s)
    good = _eng().blend_bboxes(**a, wrap=wrap)
    flipped = [t.transpose(2, 3).contiguous().transpose(2, 3) for t in a["batch_outs"]]
    assert not flipped[0].is_contiguous()
    again = _eng().blend_bboxes(**{**a, "batch_outs": flipped}, wrap=wrap)
    assert len(blend_calls) == 2 and torch.equal(_bits(good), _bits(again))
