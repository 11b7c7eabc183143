"""Every staged scatter / blend form at its capacity limit and one past it, with the launched kernel asserted.

A flag only requests a kernel form: each staged form has host-side capacity rules, and a geometry that breaks one makes
the form decline, so the call falls through to the next kernel (MultiDiffusion: row-block / strip -> TMA or cp.async ->
register-staged; the default scatter: row-block -> register-staged).  Here a CUPTI kernel trace (`launched`) records
which kernel actually ran, and every result is compared bit for bit with the torch-CPU oracle.

The geometries are literal.  Each carries the value of the metric its form is limited by, computed from the plan by a
port of the host checks (`metric`); the test recomputes the value, so a wrong port fails here, and the profiler pins
the limit itself: at the limit the requested form must launch, one past it the documented fallback must.
"""
import functools
import json
import os
import re
import tempfile
import time

import pytest
import torch

from helpers import DTYPES, assert_bit_equal, load_golden
from oracle import blend, synth, tiling

pytestmark = pytest.mark.gpu

FORCE_GENERIC, NO_TMA, TMA, PIPE, NO_PDL, ONE_PLANE, STRIP, ROWS = 1, 2, 4, 8, 32, 64, 128, 0x400

# kernel symbols of the forms
K_ASYNC, K_MOD_ASYNC, K_PIPE, K_TMA = "blend_md_async_kernel", "blend_mod_async_kernel", "blend_md_pipe_kernel", "blend_md_tma_kernel"
K_STRIP, K_STRIP_MOD = "strip_blend_kernel", "strip_blend_mod_kernel"
K_ROWS, K_ROWS_MOD, K_SCATTER_ROWS = "blend_rows_md_kernel", "blend_rows_mod_kernel", "scatter_rows_kernel"
K_VEC, K_GENERIC = "blend_grid_vec_kernel", "blend_grid_generic_kernel"
K_SCATTER_VEC, K_SCATTER_GENERIC = "scatter_vec_kernel", "scatter_generic_kernel"
KERNELS = [K_ASYNC, K_MOD_ASYNC, K_PIPE, K_TMA, K_STRIP, K_STRIP_MOD, K_ROWS, K_ROWS_MOD, K_SCATTER_ROWS, K_VEC, K_GENERIC,
           K_SCATTER_VEC, K_SCATTER_GENERIC]

# capacity constants of the host checks (csrc/td_diffusion.cu, td_strip.cu, td_rows.cu)
AS_ROWS, AS_VECS, AS_MAX_VISITS, AS_STAGE = 8, 8, 64, 1152
TMA_ROWS, TMA_VECS, TMA_MAX_VISITS, TMA_STAGE = 8, 16, 96, 2176
STAGE_BUDGET = 200 * 1024
MAX_GRID_DIM, MAX_BATCH_PTRS = 256, 128
STRIP_ROWS, STRIP_MAX_VISITS, STRIP_TABLE = 8, 64, 64 * 24
ROWS_THREADS, ROWS_MAX_COLS, ROWS_MAX_SEGS, ROWS_MAX_VEC = 512, 4, 8, 512


@pytest.fixture(scope="module")
def eng():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


# ---------------------------------------------------------------------------------------------------------------------
# which kernels ran
# ---------------------------------------------------------------------------------------------------------------------
def launched(fn) -> set:
    """Names of the CUDA kernels `fn` launches (CUPTI activity trace through torch.profiler).  Fails when the trace holds
    no kernel at all, so that a profiler without CUPTI cannot make the form assertions vacuous.

    A single session can come back incomplete: back-to-back short sessions occasionally lose an activity buffer, all of
    it (an empty trace) or part of it (the kernels launched first or last missing: every session of a call can lose
    the same leading kernels).  So each session brackets `fn` with a marker kernel (torch's spin_kernel) before and
    after it, each waited for, and counts as complete only when both markers are in its trace.  `fn`, which must be
    repeatable and launch the same kernels every time, runs in sessions until two complete ones in a row record the
    same names (at most eight sessions), and the union of what all sessions recorded is returned: a kernel counts as
    launched when any session saw it."""
    from torch.profiler import ProfilerActivity, profile
    seen, prev = set(), None
    for attempt in range(8):
        time.sleep(0.1 * attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                trace = json.load(f)
        kernels = [e.get("name", "") for e in trace.get("traceEvents", []) if e.get("cat") == "kernel"]
        names |= set(kernels)
        names.discard("")
        markers = sum("spin_kernel" in n for n in kernels)
        names = {n for n in names if "spin_kernel" not in n}
        if not names:
            continue
        seen |= names
        if markers < 2:
            continue
        if names == prev:
            break
        prev = names
    if not seen:
        raise AssertionError("the profiler recorded no CUDA kernel: the kernel-form assertions would be vacuous")
    return seen


def forms(names) -> set:
    """The project kernels among `names` (template arguments dropped)."""
    return {k for k in KERNELS for n in names if re.search(r"(?<![A-Za-z0-9_])" + k + r"(?![A-Za-z0-9_])", n)}


def template_args(names, kernel) -> list:
    out = []
    for n in names:
        m = re.search(r"(?<![A-Za-z0-9_])" + kernel + r"<([^()]*)>", n)
        if m:
            out.append([a.strip() for a in m.group(1).split(",")])
    return out


# ---------------------------------------------------------------------------------------------------------------------
# port of the host-side capacity checks, used to choose and to re-check the geometries
# ---------------------------------------------------------------------------------------------------------------------
def max_union(org, extent, size, patch):
    """max number of tiles (origins `org`, length `extent`) touching one `patch`-long block of [0, size)."""
    best = 0
    for lo in range(0, size, patch):
        hi = min(lo + patch, size) - 1
        best = max(best, sum(1 for o in org if o <= hi and o + extent > lo))
    return best


def vec_cols(xs, tw, W, vec):
    """max tile columns touching one 16-byte canvas vector (row-block forms: at most 4)."""
    return max(sum(1 for x in xs if x < (v + 1) * vec and x + tw > v * vec) for v in range(W // vec))


def rows_bands(ys, th, H, W, cols, tw, es, scatter, budget=STAGE_BUDGET):
    """rows_plan: the fewest tile-row bands per row block over the block heights it accepts otherwise (None: none)."""
    vec = 16 // es
    best = None
    for rc in range(2, 33):
        slot = segs = 0
        for b in range((H + rc - 1) // rc):
            y0, y1 = b * rc, min(H, b * rc + rc)
            nbytes = n = 0
            for y in ys:
                a, e = max(y0, y), min(y1, y + th)
                if e > a:
                    nbytes += (e - a) * cols * tw * es
                    n += 1
            slot, segs = max(slot, (y1 - y0) * W * es if scatter else nbytes), max(segs, n)
        if (not scatter and rc * (W // vec) > ROWS_THREADS) or (scatter and (tw // vec > ROWS_THREADS or rc * cols >= 16384)):
            continue
        slot = (slot + 127) & ~127
        if slot <= 0 or min(8, budget // slot) < 2:
            continue
        best = segs if best is None else min(best, segs)
    return best


def mod_rows_aux(th, tw):
    return (th * tw * 4 + 127) & ~127


class Geo:
    """A plan from engine.make_grid, checked against oracle.tiling.GridPlan, with the capacity metrics of every form."""

    def __init__(self, eng, W, H, tw, th, ov, bs):
        self.g = eng.make_grid(W, H, tw, th, ov, bs)
        self.plan = tiling.GridPlan(W, H, tw, th, ov, bs, False)
        got = [tuple(int(v) for v in r) for r in eng.grid_bboxes_xywh(self.g)]
        assert got == [tuple(b) for b in self.plan.bboxes], "engine plan differs from the oracle's"
        assert (self.g.num_batches, self.g.tile_bs) == (self.plan.num_batches, self.plan.tile_bs)
        g = self.g
        self.W, self.H, self.tw, self.th = g.W, g.H, g.tile_w, g.tile_h
        self.xs = [int(g.xs[i]) for i in range(g.cols)]
        self.ys = [int(g.ys[i]) for i in range(g.rows)]

    def metric(self, name, es):
        vec = 16 // es
        H, W, th, tw, xs, ys = self.H, self.W, self.th, self.tw, self.xs, self.ys
        if name == "as":       # cp.async MD / MoD, pipelined MD: tile visits per 8-row x 8-vector patch
            return max_union(ys, th, H, AS_ROWS) * max_union(xs, tw, W, AS_VECS * vec)
        if name == "tma":      # TMA MD: tile visits per 8-row x 16-vector patch
            return max_union(ys, th, H, TMA_ROWS) * max_union(xs, tw, W, TMA_VECS * vec)
        if name == "strip":    # strip MD / MoD: tile rows touching an 8-row strip x tile columns
            return max_union(ys, th, H, STRIP_ROWS) * len(xs)
        if name == "cols":     # row-block forms: tile columns per canvas vector
            return vec_cols(xs, tw, W, vec)
        if name == "bands":    # row-block blends: tile-row bands per row block
            return rows_bands(ys, th, H, W, len(xs), tw, es, False)
        if name == "mod_bands":
            return rows_bands(ys, th, H, W, len(xs), tw, es, False, STAGE_BUDGET - mod_rows_aux(th, tw))
        if name == "sbands":   # row-block scatter
            return rows_bands(ys, th, H, W, len(xs), tw, es, True)
        if name == "patch_rows":
            return -(-H // AS_ROWS)
        if name == "patch_cols":
            return -(-W // (AS_VECS * vec))
        if name == "row_vecs":  # row-block blend: RC * W / VEC <= 512 with RC >= 2
            return W // vec
        if name == "batches":
            return self.g.num_batches
        raise KeyError(name)

    # the dispatch of td_scatter_tiles / td_blend_multidiffusion / td_blend_mixture on this plan (tile dtype == canvas
    # dtype, aligned buffers, N * C small)
    def as_ok(self, es, mod):
        vec = 16 // es
        return (0 < self.metric("as", es) <= AS_MAX_VISITS and self.metric("patch_rows", es) <= MAX_GRID_DIM
                and self.metric("patch_cols", es) <= MAX_GRID_DIM and (not mod or self.tw % 8 == 0) and vec > 0)

    def tma_ok(self, es):
        nv = self.metric("tma", es)
        return 0 < nv <= TMA_MAX_VISITS and nv * (TMA_STAGE + 8) <= STAGE_BUDGET

    def strip_ok(self, es):
        vec = 16 // es
        xv, spv = self.W // vec, STRIP_ROWS * (self.tw // vec + 2)
        nv = self.metric("strip", es)
        nthreads = max(32, (xv * STRIP_ROWS + 31) // 32 * 32)
        return (xv * STRIP_ROWS <= 1024 and -(-self.H // STRIP_ROWS) <= MAX_GRID_DIM and 0 < nv <= STRIP_MAX_VISITS
                and nv * spv < 65536 and STRIP_TABLE + nv * spv * 16 <= STAGE_BUDGET and nv <= nthreads)

    def rows_ok(self, es, kind):
        vec = 16 // es
        if self.W // vec > ROWS_MAX_VEC or self.metric("cols", es) > ROWS_MAX_COLS:
            return False
        if kind == "mod":
            aux = mod_rows_aux(self.th, self.tw)
            if aux > STAGE_BUDGET // 2 or aux != self.th * self.tw * 4:
                return False
        b = self.metric({"md": "bands", "mod": "mod_bands", "scatter": "sbands"}[kind], es)
        return b is not None and b <= ROWS_MAX_SEGS

    def expected(self, kind, es, flags):
        vec = 16 // es
        vec_ok = not (flags & FORCE_GENERIC) and self.W % vec == 0 and self.tw % vec == 0
        if kind == "scatter":
            if not vec_ok:
                return K_SCATTER_GENERIC
            return K_SCATTER_ROWS if not (flags & NO_TMA) and self.rows_ok(es, "scatter") else K_SCATTER_VEC
        if not vec_ok:
            return K_GENERIC
        mod = kind == "mod"
        if flags & ROWS and self.rows_ok(es, kind):
            return K_ROWS_MOD if mod else K_ROWS
        if flags & STRIP and self.strip_ok(es):
            return K_STRIP_MOD if mod else K_STRIP
        if not mod and flags & TMA:
            return K_TMA if self.tma_ok(es) else K_VEC
        if not (flags & NO_TMA) and self.as_ok(es, mod):
            return K_MOD_ASYNC if mod else (K_PIPE if flags & PIPE else K_ASYNC)
        return K_VEC


# ---------------------------------------------------------------------------------------------------------------------
# one step on the device and in the oracle
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _oracle(method, dn, N, C, W, H, tw, th, ov):
    """The oracle's step; it does not depend on the tile batch size (tiles are accumulated in tile order)."""
    x = synth.latent(W * 7 + H, (N, C, H, W), DTYPES[dn])
    plan = tiling.GridPlan(W, H, tw, th, ov, 1, method == "mod")
    den = lambda t, bb: synth.fake_denoise(t, bb, N)
    if method == "md":
        return x, blend.multidiffusion_step(x, [plan.bboxes], plan.weights, den)
    return x, blend.mixture_step(x, [plan.bboxes], plan.tile_weights, plan.rescale_factor, den)


def run_blend(eng, method, dn, N, C, W, H, tw, th, ov, bs, flags, x_buffer=True, rcp=False):
    """scatter -> fake UNet per batch -> blend (profiled); returns (kernel names of the blend, bit-checked output)."""
    x, want = _oracle(method, dn, N, C, W, H, tw, th, ov)
    g = eng.make_grid(W, H, tw, th, ov, bs)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, method == "mod")
    xd = x.cuda()
    tiles = eng.scatter_tiles(g, xd)
    outs, off = [], 0
    for bbs in plan.batched_bboxes:
        outs.append(synth.fake_denoise(tiles[off * N:(off + len(bbs)) * N], bbs, N))
        off += len(bbs)
    res = {}
    if method == "md":
        w = torch.from_numpy(plan.weights).cuda()
        xb = torch.full_like(xd, float("nan")) if x_buffer else None
        r = torch.from_numpy(eng.exact_reciprocals(plan.weights)).cuda() if rcp else None
        names = launched(lambda: res.setdefault("out", eng.blend_multidiffusion(g, outs, N, C, g.tile_bs, w, xd.dtype, x_buffer=xb,
                                                                               flags=flags, rcp_weights=r)))
        out = res["out"]
        tag = f"md {dn} {(N, C, W, H, tw, th, ov, bs)} flags={flags:#x} x_buffer={x_buffer} rcp={rcp}"
        assert_bit_equal(out, want, tag)
        if x_buffer:   # x_buffer is the unnormalised accumulator: normalising it gives the output
            assert_bit_equal(blend.normalise_md(xb.cpu(), torch.from_numpy(plan.weights).view(1, 1, H, W)), want, tag + " x_buffer")
    else:
        twt = torch.from_numpy(plan.tile_weights).cuda()
        rf = torch.from_numpy(plan.rescale_factor).cuda()
        xb = torch.full_like(xd, float("nan"))
        names = launched(lambda: eng.blend_mixture(g, outs, N, C, g.tile_bs, twt, rf, xb, flags=flags))
        assert_bit_equal(xb, want, f"mod {dn} {(N, C, W, H, tw, th, ov, bs)} flags={flags:#x}")
    return names


def es_of(dn):
    return DTYPES[dn].itemsize


# ---------------------------------------------------------------------------------------------------------------------
# 1. every form at its limit and one past it
# ---------------------------------------------------------------------------------------------------------------------
# (metric, dtype family) -> ((W, H, tw, th, overlap, metric value) at the limit, (...) one past it).  The fp16 geometry
# also serves bf16 (same vector width).  No TMA geometry reaches exactly 94 visits, so 95 is the first past the limit.
# The TMA limit is 93, not kTmaMaxVisits = 96: 94+ visits need more than the 200 KB staging budget (2184 B per visit).
LIMITS = {
    ("as", "f16"): ((64, 96, 32, 32, 27, 64), (64, 64, 16, 16, 12, 65)),
    ("as", "f32"): ((64, 64, 32, 32, 28, 64), (64, 128, 48, 48, 44, 65)),
    ("tma", "f16"): ((128, 64, 8, 8, 4, 93), (128, 64, 24, 24, 18, 95)),
    ("tma", "f32"): ((128, 256, 120, 120, 116, 93), (128, 192, 80, 72, 68, 95)),
    ("strip", "f16"): ((64, 96, 32, 32, 27, 64), (96, 64, 24, 24, 18, 65)),
    ("strip", "f32"): ((64, 96, 32, 32, 27, 64), (64, 64, 16, 16, 12, 65)),
    ("cols", "f16"): ((64, 64, 8, 8, 3, 4), (64, 64, 16, 16, 11, 5)),
    ("cols", "f32"): ((64, 64, 16, 16, 11, 4), (64, 64, 24, 24, 18, 5)),
    ("bands", "f16"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
    ("bands", "f32"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
    ("mod_bands", "f16"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
    ("mod_bands", "f32"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
    ("sbands", "f16"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
    ("sbands", "f32"): ((64, 64, 40, 32, 28, 8), (64, 96, 48, 40, 35, 9)),
}

# (method, flags, metric, form at the limit, fallback past it)
FORMS = [
    ("md", 0, "as", K_ASYNC, K_VEC),
    ("md", ONE_PLANE, "as", K_ASYNC, K_VEC),
    ("md", PIPE, "as", K_PIPE, K_VEC),
    ("mod", 0, "as", K_MOD_ASYNC, K_VEC),
    ("md", TMA, "tma", K_TMA, K_VEC),
    ("md", STRIP, "strip", K_STRIP, K_ASYNC),
    ("md", STRIP | ONE_PLANE, "strip", K_STRIP, K_ASYNC),
    ("mod", STRIP, "strip", K_STRIP_MOD, K_MOD_ASYNC),
    ("md", ROWS, "cols", K_ROWS, K_ASYNC),
    ("mod", ROWS, "cols", K_ROWS_MOD, K_MOD_ASYNC),
    ("md", ROWS, "bands", K_ROWS, K_ASYNC),
    ("mod", ROWS, "mod_bands", K_ROWS_MOD, K_MOD_ASYNC),
]
LIMIT_CASES = [(m, f, met, k, fb, dn, side) for (m, f, met, k, fb) in FORMS for side in ("at", "past")
               for dn in (("f16", "bf16", "f32") if side == "at" else ("f16", "f32"))]


def _family(dn):
    return "f32" if dn == "f32" else "f16"


@pytest.mark.parametrize("method,flags,metric,kernel,fallback,dn,side", LIMIT_CASES,
                         ids=[f"{m}-{f:#x}-{met}-{dn}-{side}" for (m, f, met, _, _, dn, side) in LIMIT_CASES])
def test_blend_form_at_and_past_its_limit(eng, method, flags, metric, kernel, fallback, dn, side):
    at, past = LIMITS[(metric, _family(dn))]
    W, H, tw, th, ov, value = at if side == "at" else past
    N, C, bs = 1, 4, 4
    geo = Geo(eng, W, H, tw, th, ov, bs)
    assert geo.metric(metric, es_of(dn)) == value, "the geometry no longer has the committed metric value"
    want = kernel if side == "at" else fallback
    assert geo.expected(method, es_of(dn), flags) == want
    variants = [dict()]
    if method == "md":
        variants = [dict(x_buffer=True), dict(x_buffer=False)]
        if dn != "f32":
            variants += [dict(x_buffer=True, rcp=True)]
    for v in variants:
        names = run_blend(eng, method, dn, N, C, W, H, tw, th, ov, bs, flags, **v)
        assert forms(names) == {want}, f"{method} {metric}={value} {dn} flags={flags:#x} {v}: ran {sorted(names)}"
        if want == K_STRIP and flags & ONE_PLANE:
            assert all(a[-1] == "1" for a in template_args(names, K_STRIP)), sorted(names)


@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("side", ["at", "past"])
@pytest.mark.parametrize("metric", ["cols", "sbands"])
def test_scatter_row_block_at_and_past_its_limit(eng, metric, side, dn):
    if side == "past" and dn == "bf16":
        pytest.skip("bf16 is checked at the limit only")
    at, past = LIMITS[(metric, _family(dn))]
    W, H, tw, th, ov, value = at if side == "at" else past
    N, C = 2, 3
    geo = Geo(eng, W, H, tw, th, ov, 4)
    es = es_of(dn)
    assert geo.metric(metric, es) == value
    want = K_SCATTER_ROWS if side == "at" else K_SCATTER_VEC
    assert geo.expected("scatter", es, 0) == want
    x = synth.latent(W + 3 * H, (N, C, H, W), DTYPES[dn])
    ref = blend.scatter_tiles(x, geo.plan.bboxes)
    xd = x.cuda()
    T = geo.g.num_tiles
    for lo, hi in [(0, T), (1, T - 1), (T // 3, T // 3 + 1), (T - 2, T)]:
        res = {}
        names = launched(lambda: res.setdefault("t", eng.scatter_tiles(geo.g, xd, tile_begin=lo, tile_end=hi)))
        assert_bit_equal(res["t"], ref[lo * N:hi * N], f"scatter {metric}={value} {dn} [{lo},{hi})")
        assert forms(names) == {want}, sorted(names)


# ---------------------------------------------------------------------------------------------------------------------
# shared memory above 40 KB (the opt-in), batch tables, canvas and grid extremes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("geom,visits16", [((256, 256, 96, 96, 80), 48), ((256, 256, 32, 32, 24), 44)])
def test_cp_async_blends_above_the_shared_memory_opt_in(eng, geom, visits16, dn):
    """Ordinary UI settings on a 256 x 256 latent: 44-48 visits, 49.5-54 KB of staging in fp16 (above the 48 KB default)."""
    W, H, tw, th, ov = geom
    geo = Geo(eng, W, H, tw, th, ov, 8)
    es = es_of(dn)
    if es == 2:
        assert geo.metric("as", es) == visits16 and visits16 * AS_STAGE > 48 * 1024
    for method in ("md", "mod"):
        kernel = K_MOD_ASYNC if method == "mod" else K_ASYNC
        assert geo.expected(method, es, 0) == kernel
        names = run_blend(eng, method, dn, 1, 4, W, H, tw, th, ov, 8, 0, rcp=(method == "md" and es == 2))
        assert forms(names) == {kernel}, sorted(names)


@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("bs,batches,nb", [(27, 32, "32"), (26, 33, "128")])
def test_tma_blend_parameter_block_32_and_128_batches(eng, bs, batches, nb, dn):
    """More than 32 output tensors select the TMA kernel with 128 tensor maps (a ~16 KB __grid_constant__ block)."""
    W, H, tw, th, ov = 256, 256, 32, 32, 24
    geo = Geo(eng, W, H, tw, th, ov, bs)
    assert geo.metric("batches", es_of(dn)) == batches and geo.tma_ok(es_of(dn))
    for xb in (True, False):
        names = run_blend(eng, "md", dn, 1, 4, W, H, tw, th, ov, bs, TMA, x_buffer=xb)
        assert forms(names) == {K_TMA}, sorted(names)
        assert [a[-1] for a in template_args(names, K_TMA)] == [nb], sorted(names)


# 2056 x 16 (tile 16, overlap 8): 256 tile columns; 8 x 1028 (tile 8, overlap 4): 256 tile rows.  bs 2 -> 128 batch tensors in one launch;
# bs 1 -> 256, which the engine wrappers concatenate pairwise on the device before the launch.
GRID256 = [(2056, 16, 16, 16, 8), (8, 1028, 8, 8, 4)]


@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("geom", GRID256, ids=["256_cols", "256_rows"])
@pytest.mark.parametrize("bs", [2, 1], ids=["128_ptrs", "concat_256"])
def test_256_tile_plans_and_full_batch_tables(eng, geom, bs, dn):
    W, H, tw, th, ov = geom
    geo = Geo(eng, W, H, tw, th, ov, bs)
    assert max(geo.g.cols, geo.g.rows) == MAX_GRID_DIM
    assert geo.metric("batches", es_of(dn)) == (MAX_BATCH_PTRS if bs == 2 else 2 * MAX_BATCH_PTRS)
    es = es_of(dn)
    for method, flags in (("md", 0), ("md", TMA), ("mod", 0)):
        want = geo.expected(method, es, flags)
        names = run_blend(eng, method, dn, 1, 2, W, H, tw, th, ov, bs, flags)
        assert forms(names) == {want}, sorted(names)
        if bs == 1:   # the engine's concatenation of more than TD_MAX_BATCH_PTRS outputs ran on the device
            assert any(re.search(r"[Cc]at", n) for n in names if not forms([n])), sorted(names)
        if want == K_TMA:
            assert [a[-1] for a in template_args(names, K_TMA)] == ["128"], sorted(names)
    x = synth.latent(5, (1, 2, H, W), DTYPES[dn])
    res = {}
    names = launched(lambda: res.setdefault("t", eng.scatter_tiles(geo.g, x.cuda())))
    assert_bit_equal(res["t"], blend.scatter_tiles(x, geo.plan.bboxes), "scatter")
    assert forms(names) == {geo.expected("scatter", es, 0)}, sorted(names)


@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("H", [2048, 2056])
def test_cp_async_patch_table_height_limit(eng, H, dn):
    """256 patch rows of 8 canvas rows fill the patch tables; 2056 rows fall back to the register-staged kernel."""
    if H == 2056 and dn == "bf16":
        pytest.skip("bf16 is checked at the limit only")
    W, tw, th, ov = 64, 16, 16, 8
    geo = Geo(eng, W, H, tw, th, ov, 16)
    es = es_of(dn)
    assert geo.metric("patch_rows", es) == H // 8 and geo.g.rows <= MAX_GRID_DIM
    for method in ("md", "mod"):
        want = (K_MOD_ASYNC if method == "mod" else K_ASYNC) if H == 2048 else K_VEC
        assert geo.expected(method, es, 0) == want
        names = run_blend(eng, method, dn, 1, 1, W, H, tw, th, ov, 16, 0)
        assert forms(names) == {want}, sorted(names)


@pytest.mark.parametrize("dn", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("side", ["at", "past"])
def test_row_block_blend_width_limit(eng, side, dn):
    """RC * W / VEC <= 512 with RC >= 2: W = 2048 (fp16) / 1024 (fp32) is the widest row-block canvas."""
    if side == "past" and dn == "bf16":
        pytest.skip("bf16 is checked at the limit only")
    es = es_of(dn)
    W = (2048 if es == 2 else 1024) + (0 if side == "at" else 8)
    H, tw, th, ov = 16, 16, 16, 8
    geo = Geo(eng, W, H, tw, th, ov, 32)
    assert geo.metric("row_vecs", es) == W // (16 // es)
    for method in ("md", "mod"):
        want = (K_ROWS_MOD if method == "mod" else K_ROWS) if side == "at" else (K_MOD_ASYNC if method == "mod" else K_ASYNC)
        assert geo.expected(method, es, ROWS) == want
        names = run_blend(eng, method, dn, 1, 1, W, H, tw, th, ov, 32, ROWS)
        assert forms(names) == {want}, sorted(names)


# ---------------------------------------------------------------------------------------------------------------------
# 2. which form the existing parametrizations run
# ---------------------------------------------------------------------------------------------------------------------
ALL_PATHS = [0, NO_PDL, ROWS, ROWS | NO_PDL, ONE_PLANE, PIPE, TMA, NO_TMA, FORCE_GENERIC, STRIP, STRIP | ONE_PLANE]
EDGE_CASES = [  # test_gpu_diffusion.test_blend_vs_oracle_edge_geometries
    (1, 4, 96, 96, 96, 96, 48, 4), (2, 4, 40, 30, 96, 96, 48, 4), (2, 4, 97, 96, 96, 96, 48, 4), (1, 4, 200, 8, 16, 8, 12, 7),
    (2, 4, 8, 200, 8, 16, 12, 5), (1, 1, 104, 104, 24, 24, 20, 16), (2, 4, 768, 768, 128, 128, 64, 8),
]
SCATTER_CASES = [  # test_gpu_diffusion.test_scatter_bit_exact
    (2, 4, 64, 48, 16, 16, 8), (1, 4, 57, 43, 16, 16, 12), (2, 4, 128, 128, 96, 96, 48), (3, 5, 96, 64, 40, 24, 4),
    (2, 4, 512, 512, 96, 96, 48), (1, 9, 72, 72, 24, 16, 6), (2, 4, 100, 77, 32, 24, 8),
]
# the form a flag requests (flags not listed request the default cp.async form)
REQUESTED = {("md", ROWS): K_ROWS, ("md", ROWS | NO_PDL): K_ROWS, ("md", PIPE): K_PIPE, ("md", TMA): K_TMA, ("md", NO_TMA): K_VEC,
             ("md", FORCE_GENERIC): K_GENERIC, ("md", STRIP): K_STRIP, ("md", STRIP | ONE_PLANE): K_STRIP,
             ("mod", ROWS): K_ROWS_MOD, ("mod", ROWS | NO_PDL): K_ROWS_MOD, ("mod", NO_TMA): K_VEC, ("mod", FORCE_GENERIC): K_GENERIC,
             ("mod", STRIP): K_STRIP_MOD, ("mod", STRIP | ONE_PLANE): K_STRIP_MOD}
# (fixture set, case, method, dtype family) -> {flags: kernel} wherever a flag does not get the form it requests
FALLBACKS = {
    ("edge", (2, 4, 40, 30, 96, 96, 48, 4), "mod", "f16"): {ROWS: K_MOD_ASYNC, ROWS | NO_PDL: K_MOD_ASYNC},
    ("edge", (2, 4, 40, 30, 96, 96, 48, 4), "mod", "f32"): {ROWS: K_MOD_ASYNC, ROWS | NO_PDL: K_MOD_ASYNC},
}


def test_existing_parametrizations_run_the_forms_they_request(eng, golden_dir):
    """Replays the geometries of test_blend_small_matches_reference_fixtures, test_blend_vs_oracle_edge_geometries and
    test_scatter_bit_exact: each (case, dtype, flags) must run the kernel the host checks choose, the 40 x 30 MoD ROWS
    fallback included, and every requested form must run on at least one case per dtype, so that a change to a limit
    cannot empty a parametrization unnoticed."""
    g = load_golden(golden_dir, "blend_small")
    small = [tuple(int(v) for v in c) for c in g["cases"]]
    seen = {}
    for name, cases, dtypes in (("small", small, ("f16", "bf16", "f32")), ("edge", EDGE_CASES, ("f16", "f32"))):
        for case in cases:
            N, C, W, H, tw, th, ov, bs = case
            geo = Geo(eng, W, H, tw, th, ov, bs)
            for dn in dtypes:
                es = es_of(dn)
                x = synth.latent(3, (N, C, H, W), DTYPES[dn]).cuda()
                tiles = eng.scatter_tiles(geo.g, x)
                outs = [tiles]
                for method in ("md", "mod"):
                    fb = FALLBACKS.get((name, case, method, _family(dn)), {})
                    for flags in ALL_PATHS:
                        want = geo.expected(method, es, flags)
                        if flags in fb:
                            assert want == fb[flags], (name, case, method, dn, flags)
                        if method == "md":
                            w = torch.from_numpy(geo.plan.weights).cuda()
                            fn = lambda: eng.blend_multidiffusion(geo.g, outs, N, C, geo.g.num_tiles, w, x.dtype, flags=flags)
                        else:
                            p = tiling.GridPlan(W, H, tw, th, ov, bs, True)
                            twt, rf = torch.from_numpy(p.tile_weights).cuda(), torch.from_numpy(p.rescale_factor).cuda()
                            xb = torch.empty_like(x)
                            fn = lambda: eng.blend_mixture(geo.g, outs, N, C, geo.g.num_tiles, twt, rf, xb, flags=flags)
                        got = forms(launched(fn))
                        assert got == {want}, f"{name} {case} {method} {dn} flags={flags:#x}: ran {sorted(got)}, expected {want}"
                        seen.setdefault((method, dn, flags), set()).add(want)
    for (method, dn, flags), ks in seen.items():
        req = REQUESTED.get((method, flags), K_MOD_ASYNC if method == "mod" else K_ASYNC)
        assert req in ks, f"{method} {dn} flags={flags:#x}: no case runs {req} (ran {sorted(ks)})"
    for case in SCATTER_CASES:
        N, C, W, H, tw, th, ov = case
        geo = Geo(eng, W, H, tw, th, ov, 4)
        for dn in DTYPES:
            x = synth.latent(7, (N, C, H, W), DTYPES[dn]).cuda()
            for flags in (0, NO_TMA, FORCE_GENERIC):
                got = forms(launched(lambda: eng.scatter_tiles(geo.g, x, flags=flags)))
                assert got == {geo.expected("scatter", es_of(dn), flags)}, f"scatter {case} {dn} flags={flags:#x}: ran {sorted(got)}"
                seen.setdefault(("scatter", dn, flags), set()).update(got)
    for dn in DTYPES:
        assert K_SCATTER_ROWS in seen[("scatter", dn, 0)] and K_SCATTER_VEC in seen[("scatter", dn, NO_TMA)]
