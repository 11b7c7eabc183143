"""The inpaint sparse blends and the SpotDiffusion step plans at every kernel form and staging limit, bit for bit against
CPU oracles, with the kernel that ran asserted.

Sparse blends (td_blend_multidiffusion_sparse / td_blend_mixture_sparse) are compared with tests/sparse_oracle.py -- the
kept tiles added in tile order with the full plan's weights -- at the cp.async visit limit and one past it, with visit
tables that span all three warps of a CTA, on every route to the generic kernel (odd widths, each misaligned pointer,
mixed dtypes, more than 256 patch rows, TD_FLAG_FORCE_GENERIC), with permuted slot tables, empty / single / full active
sets, more than 128 compact batches and a 65536-tile plan.  `SPARSE_FORM_MATRIX` lists every sparse instantiation an
entry can launch; one test launches them all.  td_grid_active_tiles is pinned at the values next to 1.0, signed zeros,
infinities, subnormals and NaN, against the rule of tests/test_inpaint_mask_plan.py.

SpotDiffusion's step plans (td_grid_shift) crowd windows at both ends of a bounded axis, so a step plan can hold more
visits per cp.async patch than its base plan: at 128 / 112 on a 256^2 latent the base plan runs the cp.async blend (64
visits) and every step plan the register-staged one (81).  The scatter and blend of step plans at the sizes the UI
reaches are compared with tests/spot_oracle.py, and the kernel the port of the host checks predicts must run.

The CPU part (no mark) checks the oracle against oracle/blend.py, shows that the bit checks catch a visit table with a
dropped, a reordered or a skipped tile's visit, pins the visit counts the geometries claim, and compares the form matrix
with the kernels a cubin build of td_diffusion.cu holds.

The file name sorts it after every GPU test file that reads a kernel trace in the main pytest process (the last is
test_gpu_vae_kernels.py).  Such traces lose kernel records once the process has run long enough.  This file adds about
200 s to the process: its bit checks, plus the wait for its fresh-interpreter rerun.  Run before test_gpu_vae_kernels.py
in a full GPU suite, it pushes that file's trace past the point where records go missing.
"""
import ctypes
import os
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

import sparse_oracle as spo
import spot_oracle as so
import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal
from oracle import blend, synth, tiling
from test_gpu_blend_limits import (AS_MAX_VISITS, K_ASYNC, K_GENERIC, K_MOD_ASYNC, K_SCATTER_GENERIC, K_SCATTER_ROWS,
                                   K_SCATTER_VEC, K_VEC, LIMITS, Geo, forms, launched, template_args)
from test_inpaint_mask_plan import JUST_BELOW_ONE, rule

gpu = pytest.mark.gpu

FORCE_GENERIC, NO_PDL, ONE_PLANE = 1, 32, 64
CT = {"f16": "__half", "bf16": "__nv_bfloat16", "f32": "float"}   # template argument spelling of each dtype
MODE = {"md": "0", "mod": "1"}
SPARSE_KERNELS = (K_ASYNC, K_MOD_ASYNC, K_GENERIC)


def _eng():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def es_of(dn):
    return DTYPES[dn].itemsize


# ---------------------------------------------------------------------------------------------------------------------
# the sparse instantiations
# ---------------------------------------------------------------------------------------------------------------------
def async_form(dn, x_buffer, rcp):
    """blend_md_async_kernel<T, WRITE_BUF, FASTDIV, 1, true>: FASTDIV only for 16-bit tiles given rcp_weights."""
    fd = rcp and dn != "f32"
    return (K_ASYNC, (CT[dn], "true" if x_buffer else "false", "true" if fd else "false", "1", "true"))


def mod_async_form(dn):
    return (K_MOD_ASYNC, (CT[dn], "false", "true"))


def generic_form(method, tile_dn, acc_dn):
    return (K_GENERIC, (CT[tile_dn], CT[acc_dn], MODE[method], "true"))


# Every sparse instantiation an entry can launch: 10 MultiDiffusion cp.async (FASTDIV needs a 16-bit tile: the fp32
# <float, *, true, 1, true> pair is compiled, since the FASTDIV choice is made at run time, but no call reaches it),
# 3 Mixture of Diffusers cp.async, and the generic kernel at the 9 tile / accumulator dtype pairs of both methods.
SPARSE_FORM_MATRIX = sorted(
    {async_form(dn, xb, rcp) for dn in DTYPES for xb in (False, True) for rcp in (False, True)}
    | {mod_async_form(dn) for dn in DTYPES}
    | {generic_form(m, t, a) for m in MODE for t in DTYPES for a in DTYPES})
UNREACHABLE = [(K_ASYNC, ("float", "false", "true", "1", "true")), (K_ASYNC, ("float", "true", "true", "1", "true"))]


def test_sparse_form_matrix_lists_31_forms():
    assert len(SPARSE_FORM_MATRIX) == 31
    assert sum(k == K_ASYNC for k, _ in SPARSE_FORM_MATRIX) == 10 and sum(k == K_GENERIC for k, _ in SPARSE_FORM_MATRIX) == 18
    assert not set(UNREACHABLE) & set(SPARSE_FORM_MATRIX)


NVCC = "/usr/local/cuda/bin/nvcc"


@pytest.mark.skipif(not (os.path.exists(NVCC) and shutil.which("c++filt")), reason="needs nvcc and c++filt")
def test_sparse_form_matrix_is_every_compiled_sparse_kernel():
    """The sparse kernels of a cubin build of td_diffusion.cu (no GPU needed) are the matrix plus the two unreachable
    fp32 FASTDIV ones."""
    saved = list(sys.path)
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "debug_tools"))
    try:
        import sass_identity as si          # puts the package directory on sys.path to read its nvcc flags
    finally:
        sys.path[:] = saved
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "td_diffusion.cubin")
        si.compile_cubin(os.path.join(si.ROOT, si.SRC), cubin)
        names = list(si.functions(cubin))
    found = set()
    for n in si.demangle(names).values():
        for k in SPARSE_KERNELS:
            for a in template_args([n], k):
                if a[-1] == "true":
                    found.add((k, tuple(a)))
    assert found == set(SPARSE_FORM_MATRIX) | set(UNREACHABLE), (sorted(set(SPARSE_FORM_MATRIX) - found), sorted(found - set(SPARSE_FORM_MATRIX)))


# ---------------------------------------------------------------------------------------------------------------------
# which kernel ran: asserted in a fresh interpreter (CUPTI traces are reliable only in a young process, see
# tests/test_gpu_wrap_forms.py); elsewhere `_traced` only runs the call.  Every bit check runs in both.
# ---------------------------------------------------------------------------------------------------------------------
FORMS_CHILD = os.environ.get("TD_SPARSE_SPOT_FORMS_CHILD") == "1"
FORM_TESTS = "not fresh_process and not delegate"


def _traced(fn, kernels=SPARSE_KERNELS):
    """{(kernel, template arguments)} of the `kernels` fn launched (child interpreter), or None after running it."""
    if not FORMS_CHILD:
        fn()
        return None
    names = launched(fn)
    return {(k, tuple(a)) for k in kernels for a in template_args(names, k)}, names


def _assert_form(traced, want, what):
    if traced is None:
        return
    got, names = traced
    assert got == {want}, f"{what}: ran {sorted(got)} ({sorted(names)}), expected {want}"


@gpu
def test_launched_forms_in_a_fresh_process():
    """The GPU tests rerun in a fresh interpreter, where they also assert which kernel form ran."""
    if FORMS_CHILD:
        pytest.skip("already the child interpreter")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    cmd = [sys.executable, *flags, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k", FORM_TESTS]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(cmd, cwd=root, env=dict(os.environ, TD_SPARSE_SPOT_FORMS_CHILD="1"), capture_output=True, text=True, timeout=2400)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail


# ---------------------------------------------------------------------------------------------------------------------
# a plan, the full plan's tile outputs, and one sparse blend against the oracle
# ---------------------------------------------------------------------------------------------------------------------
class Job:
    """A make_grid plan (checked against oracle.tiling by Geo), its MultiDiffusion weights, Mixture of Diffusers tile weights
    and rescale factor, and an output for every tile in tile order."""

    def __init__(self, W, H, tw, th, ov, bs, N=1, C=2, seed=0):
        self.geo = Geo(_eng(), W, H, tw, th, ov, bs)
        self.g = self.geo.g
        self.N, self.C, self.T = N, C, self.g.num_tiles
        self.bboxes = [tuple(b) for b in self.geo.plan.bboxes]
        self.weights = self.geo.plan.weights
        mod = tiling.GridPlan(W, H, tw, th, ov, bs, True)
        self.tile_weights, self.rescale = mod.tile_weights, mod.rescale_factor
        assert np.isfinite(self.rescale).all()
        self.seed = seed
        self._tiles = {}

    def tiles(self, dn):
        if dn not in self._tiles:
            gen = torch.Generator().manual_seed(self.seed + 31 * self.T)
            t = torch.randn((self.T * self.N, self.C, self.geo.th, self.geo.tw), generator=gen) * 2
            self._tiles[dn] = t.to(DTYPES[dn])
        return self._tiles[dn]

    def want(self, method, active, tile_dn, acc_dn):
        if method == "md":
            return spo.sparse_md(self.tiles(tile_dn), self.bboxes, active, self.N, self.weights, DTYPES[acc_dn])
        return spo.sparse_mod(self.tiles(tile_dn), self.bboxes, active, self.N, self.tile_weights, self.rescale, DTYPES[acc_dn])

    def tables(self, es):
        return spo.patch_tables(self.geo.xs, self.geo.ys, self.geo.tw, self.geo.th, self.geo.W, self.geo.H, es)


def _shifted(t):
    """A copy of `t` one element past a 16-byte boundary (an offset view into a larger buffer)."""
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def _nan(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def _slots(active, perm_seed=None):
    """The slot table of `active` (monotone, or a random permutation of the positions) and the kept tiles by position."""
    slot = _eng().slot_table(active)
    kept = np.flatnonzero(active)
    if perm_seed is not None and len(kept) > 1:
        pos = np.random.default_rng(perm_seed).permutation(len(kept)).astype(np.int32)
        slot[kept] = pos
        order = np.empty(len(kept), dtype=np.int64)
        order[pos] = kept
        kept = order
    return slot, kept


def run_sparse(job, method, active, acc_dn, tile_dn=None, x_buffer=True, rcp=False, shift=(), flags=0, perm_seed=None,
               tile_bs=None):
    """One sparse blend through the C ABI (every pointer under the test's control), checked bit for bit against the oracle.
    Returns what `_traced` returns."""
    cabi, lib = _cabi(), _cabi().lib
    tile_dn = tile_dn or acc_dn
    N, C, g = job.N, job.C, job.g
    acc = DTYPES[acc_dn]
    slot, order = _slots(active, perm_seed)
    K = len(order)
    bs = tile_bs or g.tile_bs
    tiles = job.tiles(tile_dn)
    compact = tiles.view(job.T, N, C, g.tile_h, g.tile_w)[torch.from_numpy(order)].reshape(K * N, C, g.tile_h, g.tile_w)
    batches = [compact[i * N:min(i + bs, K) * N].cuda() for i in range(0, K, bs)]
    if "tiles" in shift and batches:
        batches[-1] = _shifted(batches[-1])
    assert len(batches) <= cabi.TD_MAX_BATCH_PTRS
    ptrs = (ctypes.c_void_p * max(1, len(batches)))(*[b.data_ptr() for b in batches])
    slot_dev = torch.from_numpy(slot).cuda()
    slot_ptr = slot.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
    stream = cabi.current_stream_ptr()
    tag = f"{method} tile={tile_dn} acc={acc_dn} {(g.W, g.H, g.tile_w, g.tile_h)} K={K}/{job.T} x_buffer={x_buffer} rcp={rcp} shift={shift} flags={flags:#x} perm={perm_seed}"
    if method == "md":
        want_out, want_buf = job.want("md", active, tile_dn, acc_dn)
        w = torch.from_numpy(job.weights).cuda()
        w = _shifted(w) if "weights" in shift else w
        r = torch.from_numpy(_eng().exact_reciprocals(job.weights)).cuda() if rcp else None
        r = _shifted(r) if r is not None and "rcp" in shift else r
        xo = _nan((N, C, g.H, g.W), torch.float32)
        xo = _shifted(xo) if "x_out" in shift else xo
        xb = _nan((N, C, g.H, g.W), acc) if x_buffer else None
        xb = _shifted(xb) if xb is not None and "x_buffer" in shift else xb

        def call():
            rc = lib.td_blend_multidiffusion_sparse(ctypes.byref(g), ptrs, len(batches), bs, N, C, cabi.dtype_code(DTYPES[tile_dn]),
                                                    cabi.dtype_code(acc), w.data_ptr(), r.data_ptr() if r is not None else None,
                                                    xo.data_ptr(), xb.data_ptr() if xb is not None else None, slot_dev.data_ptr(),
                                                    slot_ptr, job.T, flags, stream)
            assert rc == cabi.TD_OK, (tag, lib.td_last_error())
        traced = _traced(call)
        torch.cuda.synchronize()
        assert_bit_equal(xo.cpu(), want_out, tag)
        if xb is not None:
            assert_bit_equal(xb.cpu(), want_buf, tag + " x_buffer")
        return traced
    want = job.want("mod", active, tile_dn, acc_dn)
    twt = torch.from_numpy(job.tile_weights).cuda()
    twt = _shifted(twt) if "tile_weights" in shift else twt
    rs = torch.from_numpy(job.rescale).cuda()
    rs = _shifted(rs) if "rescale" in shift else rs
    xb = _nan((N, C, g.H, g.W), acc)
    xb = _shifted(xb) if "x_buffer" in shift else xb

    def call():
        rc = lib.td_blend_mixture_sparse(ctypes.byref(g), ptrs, len(batches), bs, N, C, cabi.dtype_code(DTYPES[tile_dn]), cabi.dtype_code(acc),
                                         twt.data_ptr(), rs.data_ptr(), xb.data_ptr(), slot_dev.data_ptr(), slot_ptr, job.T, flags, stream)
        assert rc == cabi.TD_OK, (tag, lib.td_last_error())
    traced = _traced(call)
    torch.cuda.synchronize()
    assert_bit_equal(xb.cpu(), want, tag)
    return traced


def expected_form(job, method, acc_dn, tile_dn=None, x_buffer=True, rcp=False, shift=(), flags=0):
    """The port of the sparse entries' dispatch: the cp.async kernel when the vector conditions and its capacity rules hold,
    else the generic one."""
    tile_dn = tile_dn or acc_dn
    es = es_of(tile_dn)
    vec = 16 // es
    checked = {"md": ("tiles", "weights", "rcp", "x_out", "x_buffer"), "mod": ("tiles", "rescale", "x_buffer")}[method]
    vec_ok = (not flags & FORCE_GENERIC and tile_dn == acc_dn and job.geo.W % vec == 0 and job.geo.tw % vec == 0
              and not set(shift) & set(checked))
    if method == "mod" and "tile_weights" in shift:
        vec_ok = False          # the cp.async MoD kernel reads the tile weights with 16-byte loads
    if vec_ok and job.geo.as_ok(es, method == "mod"):
        return async_form(acc_dn, x_buffer, rcp) if method == "md" else mod_async_form(acc_dn)
    return generic_form(method, tile_dn, acc_dn)


def high_positions(job, es):
    """Only the visits at positions >= 32 of the fullest patch's table: they land in the second and third warps of the CTA,
    so every one of them is placed by the cross-warp prefix of prepare_sparse_visits."""
    tables = job.tables(es)
    table = tables[spo.fullest_patch(tables)][1]
    assert len(table) == job.geo.metric("as", es) > 32, "the fullest patch must span more than one warp"
    active = np.zeros(job.T, bool)
    active[table[32:]] = True
    return active


def active_sets(job, es, seed=0):
    T = job.T
    out = {"all": np.ones(T, bool), "none": np.zeros(T, bool), "first": np.arange(T) == 0, "last": np.arange(T) == T - 1,
           "alternate": np.arange(T) % 2 == 0, "random40": np.random.default_rng(seed + T).random(T) < 0.4}
    if job.geo.metric("as", es) > 32:
        out["high_positions"] = high_positions(job, es)
    return out


def _family(dn):
    return "f32" if dn == "f32" else "f16"


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle and the defects its checks catch
# ---------------------------------------------------------------------------------------------------------------------
def _cpu_plan(W, H, tw, th, ov, N=1, C=2, dn="f16", seed=0):
    md, mod = tiling.GridPlan(W, H, tw, th, ov, 4, False), tiling.GridPlan(W, H, tw, th, ov, 4, True)
    T = len(md.bboxes)
    tiles = (torch.randn((T * N, C, th, tw), generator=torch.Generator().manual_seed(seed)) * 2).to(DTYPES[dn])
    xs = sorted({b[0] for b in md.bboxes})
    ys = sorted({b[1] for b in md.bboxes})
    return md, mod, tiles, xs, ys


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("method", ["md", "mod"])
def test_oracle_with_every_tile_kept_is_the_dense_oracle(method, dn):
    W, H, tw, th, ov, N = 100, 72, 32, 24, 12, 2
    md, mod, tiles, _, _ = _cpu_plan(W, H, tw, th, ov, N=N, dn=dn)
    T = len(md.bboxes)
    x = torch.zeros((N, 2, H, W), dtype=DTYPES[dn])
    den = lambda t, bb: tiles                                         # noqa: E731  (one batch: the whole plan)
    everything = np.ones(T, bool)
    if method == "md":
        got, _ = spo.sparse_md(tiles, md.bboxes, everything, N, md.weights, DTYPES[dn])
        assert_bit_equal(got, blend.multidiffusion_step(x, [md.bboxes], md.weights, den), "md")
    else:
        got = spo.sparse_mod(tiles, mod.bboxes, everything, N, mod.tile_weights, mod.rescale_factor, DTYPES[dn])
        assert_bit_equal(got, blend.mixture_step(x, [mod.bboxes], mod.tile_weights, mod.rescale_factor, den), "mod")


@pytest.mark.parametrize("method", ["md", "mod"])
def test_oracle_leaves_uncovered_pixels_at_positive_zero(method):
    W, H, tw, th, ov = 100, 72, 32, 24, 12
    md, mod, tiles, _, _ = _cpu_plan(W, H, tw, th, ov)
    T = len(md.bboxes)
    active = np.random.default_rng(1).random(T) < 0.3
    cover = torch.zeros((H, W), dtype=torch.int32)
    for t in np.flatnonzero(active):
        x, y, w, h = md.bboxes[t]
        cover[y:y + h, x:x + w] += 1
    assert (cover == 0).any() and (cover > 0).any()
    if method == "md":
        outs = spo.sparse_md(tiles, md.bboxes, active, 1, md.weights, torch.float16)
    else:
        outs = (spo.sparse_mod(tiles, mod.bboxes, active, 1, mod.tile_weights, mod.rescale_factor, torch.float16),)
    for o in outs:
        z = (cover == 0).expand_as(o)
        assert_bit_equal(o[z], torch.zeros_like(o[z]), "uncovered pixels are +0")


def _defect_case(kind, method):
    """(plan pieces, tiles, active, defect): the 64-visit fp16 geometry of LIMITS, every visit of the fullest patch kept
    except for the skipped-tile defect."""
    W, H, tw, th, ov, visits = LIMITS[("as", "f16")][0]
    md, mod, tiles, xs, ys = _cpu_plan(W, H, tw, th, ov, dn="f16", seed=3)
    T = len(md.bboxes)
    tables = spo.patch_tables(xs, ys, tw, th, W, H, 2)
    p = spo.fullest_patch(tables)
    table = tables[p][1]
    assert len(table) == visits
    active = np.ones(T, bool)
    if kind == "drop":
        return md, mod, tiles, xs, ys, active, ("drop", p, 45)
    if kind == "include":
        active = np.random.default_rng(2).random(T) < 0.5
        skipped = [t for t in table if not active[t]]
        return md, mod, tiles, xs, ys, active, ("include", p, skipped[len(skipped) // 2])
    # swap: three visits sharing a pixel of the patch, values whose fp16 sum depends on the order of the last two:
    # (1 + 2^-11) rounds to 1 (a tie, to even), so 1 + 2^-11 - 1 = 0, while 1 - 1 + 2^-11 = 2^-11
    (x0, y0, x1, y1), _ = tables[p]
    cols = len(xs)
    k, i, j = table[0], table[1], table[2]
    boxes = [(xs[t % cols], ys[t // cols]) for t in (k, i, j)]
    px, py = max([x0] + [b[0] for b in boxes]), max([y0] + [b[1] for b in boxes])
    assert x0 <= px < x1 and y0 <= py < y1 and all(bx + tw > px and by + th > py for bx, by in boxes)
    tiles = torch.zeros_like(tiles)
    scale = 1.0 if method == "md" else 1.0 / float(mod.tile_weights[py - boxes[0][1], px - boxes[0][0]] * mod.rescale_factor[py, px])
    for t, v in ((k, 1.0), (i, 2.0 ** -11), (j, -1.0)):
        tiles[t] = v if method == "md" else v * scale
    return md, mod, tiles, xs, ys, active, ("swap", p, 1, 2)


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("kind", ["drop", "swap", "include"])
def test_checks_catch_injected_visit_table_defects(kind, method):
    """The CPU model of the cp.async visit table gives the oracle's bits, and each defect in one patch's table fails the
    same bit check the GPU tests apply."""
    md, mod, tiles, xs, ys, active, defect = _defect_case(kind, method)
    tw, th = md.tile_w, md.tile_h
    if method == "md":
        want = spo.sparse_md(tiles, md.bboxes, active, 1, md.weights, torch.float16)
        run = lambda d: spo.emulate("md", tiles, xs, ys, tw, th, active, 1, torch.float16, 2, weights=md.weights, defect=d)  # noqa: E731
    else:
        want = (spo.sparse_mod(tiles, mod.bboxes, active, 1, mod.tile_weights, mod.rescale_factor, torch.float16),)
        run = lambda d: (spo.emulate("mod", tiles, xs, ys, tw, th, active, 1, torch.float16, 2, tile_weights=mod.tile_weights,  # noqa: E731
                                     rescale=mod.rescale_factor, defect=d),)
    for got, w in zip(run(None), want):
        assert_bit_equal(got, w, "the visit-table model without a defect")
    bad = run(defect)
    with pytest.raises(AssertionError):
        assert_bit_equal(bad[0], want[0], kind)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the visit counts the geometries claim (port of the host checks, on engine plans)
# ---------------------------------------------------------------------------------------------------------------------
UI = [((256, 256, 96, 96, 80), 48), ((256, 256, 32, 32, 24), 44)]   # (geometry, fp16 visits of the fullest patch)


@pytest.mark.parametrize("geom,visits", UI)
def test_ui_geometries_fill_more_than_one_warp(geom, visits):
    geo = Geo(_eng(), *geom, 8)
    assert geo.metric("as", 2) == visits > 32 and geo.as_ok(2, False) and geo.as_ok(2, True)
    assert geo.as_ok(4, False) and geo.as_ok(4, True)


class SpotGeo(Geo):
    """A SpotDiffusion step plan from engine.shift_grid, with its bboxes checked against spot_oracle.SpotPlan, and the
    capacity metrics of Geo."""

    def __init__(self, eng, W, H, tw, th, ov, bs, wrap, sx, sy):
        base = eng.make_grid(W, H, tw, th, ov, bs, wrap=wrap)
        self.base = base
        self.g = g = eng.shift_grid(base, sx, sy, bs)
        self.plan = so.SpotPlan(W, H, tw, th, ov, bs, wrap, sx, sy)
        got = [tuple(int(v) for v in r) for r in eng.grid_bboxes_xywh(g)]
        assert got == self.plan.bboxes, "engine step plan differs from the oracle's"
        assert (g.num_batches, g.tile_bs) == (self.plan.num_batches, self.plan.tile_bs)
        self.W, self.H, self.tw, self.th = g.W, g.H, g.tile_w, g.tile_h
        self.xs = [int(g.xs[i]) for i in range(g.cols)]
        self.ys = [int(g.ys[i]) for i in range(g.rows)]


def _shifts(W, H, tw, th, ov, wrap):
    lo_x, hi_x, lo_y, hi_y = so.bounds(W, H, tw, th, ov, wrap)
    return sorted({(lo_x, lo_y), ((lo_x + hi_x) // 2, (lo_y + hi_y) // 2), (hi_x - 1, hi_y - 1)})


# (W, H, tile, overlap, wrap) of the step-plan tests; the 256^2 ones cross a visit limit between base and step plans
CFG2 = [(512, 512, 96, ov, 0) for ov in (0, 8, 48)]
PANORAMA = [(2048, 512, 96, 8, 0), (2048, 512, 96, 8, so.WRAP_X)]
CROSSING = {(256, 256, 128, 112, 0): (64, (81, 81)), (256, 256, 64, 52, 0): (60, (66, 77)), (256, 256, 96, 72, 0): (30, (35, 42))}
SPOT_GEOMS = CFG2 + PANORAMA + list(CROSSING)


@pytest.mark.parametrize("geom", list(CROSSING), ids=[f"{g[2]}_{g[3]}" for g in CROSSING])
def test_step_plans_hold_more_visits_than_their_base_plan(geom):
    """fp16 visits per cp.async patch: the base plan's, and the range over the lowest, middle and highest shift."""
    W, H, t, ov, wrap = geom
    base_visits, (lo, hi) = CROSSING[geom]
    eng = _eng()
    assert Geo(eng, W, H, t, t, ov, 8).metric("as", 2) == base_visits
    got = [SpotGeo(eng, W, H, t, t, ov, 8, wrap, sx, sy).metric("as", 2) for sx, sy in _shifts(W, H, t, t, ov, wrap)]
    assert lo <= min(got) and max(got) <= hi and max(got) > base_visits, got
    if t == 128:
        assert base_visits == AS_MAX_VISITS and min(got) > AS_MAX_VISITS     # cp.async on the base plan, vector on every step plan


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every sparse instantiation
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_every_sparse_instantiation_launches():
    """Each entry of SPARSE_FORM_MATRIX launches on some call, bit-equal to the oracle, and no other sparse form does."""
    job = Job(256, 136, 64, 64, 24, 3, N=2, C=2)
    active = np.random.default_rng(4).random(job.T) < 0.6
    seen = set()

    def add(traced, want):
        _assert_form(traced, want, "")
        if traced is not None:
            seen.update(traced[0])
    for dn in DTYPES:
        for xb in (False, True):
            for rcp in (False, True):
                add(run_sparse(job, "md", active, dn, x_buffer=xb, rcp=rcp), async_form(dn, xb, rcp))
        add(run_sparse(job, "mod", active, dn), mod_async_form(dn))
        for tile_dn in DTYPES:
            for method in ("md", "mod"):
                flags = FORCE_GENERIC if tile_dn == dn else 0
                add(run_sparse(job, method, active, dn, tile_dn=tile_dn, flags=flags), generic_form(method, tile_dn, dn))
    if FORMS_CHILD:
        assert seen == set(SPARSE_FORM_MATRIX), f"missing {sorted(set(SPARSE_FORM_MATRIX) - seen)}, unlisted {sorted(seen - set(SPARSE_FORM_MATRIX))}"
        print(f"all {len(SPARSE_FORM_MATRIX)} entries of SPARSE_FORM_MATRIX launched")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the cp.async visit limit, visit tables across warps
# ---------------------------------------------------------------------------------------------------------------------
def _md_variants(dn):
    """(x_buffer, rcp): the forms the delegates use -- rcp_weights without x_buffer is the fp16 / bf16 inpaint default."""
    return [(True, False), (False, False), (False, True), (True, True)] if dn != "f32" else [(True, False), (False, False)]


@gpu
@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("side", ["at", "past"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_sparse_blend_at_and_past_the_visit_limit(dn, side, method):
    """64 visits run the sparse cp.async kernel; 65 the sparse generic one (the sparse entries have no register-staged form)."""
    at, past = LIMITS[("as", _family(dn))]
    W, H, tw, th, ov, visits = at if side == "at" else past
    job = Job(W, H, tw, th, ov, 4, N=1, C=3)
    es = es_of(dn)
    assert job.geo.metric("as", es) == visits
    for name, active in active_sets(job, es).items():
        for xb, rcp in (_md_variants(dn) if method == "md" else [(True, False)]):
            want = expected_form(job, method, dn, x_buffer=xb, rcp=rcp)
            if side == "past":
                assert want == generic_form(method, dn, dn)
            else:
                assert want[0] == (K_ASYNC if method == "md" else K_MOD_ASYNC)
            _assert_form(run_sparse(job, method, active, dn, x_buffer=xb, rcp=rcp), want, f"{name} {side} {dn} {method} {xb} {rcp}")


@gpu
@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("geom,visits", UI, ids=["96_80", "32_24"])
def test_sparse_blend_ui_geometries(geom, visits, dn, method):
    """Ordinary UI settings on a 256^2 latent: 44-48 visits per fp16 patch, so the kept visits of a patch span all three
    warps of the CTA."""
    job = Job(*geom, 8, N=1, C=2)
    es = es_of(dn)
    if es == 2:
        assert job.geo.metric("as", es) == visits > 32
    for name, active in active_sets(job, es, seed=9).items():
        for xb, rcp in (_md_variants(dn)[1:3] if method == "md" else [(True, False)]):
            want = expected_form(job, method, dn, x_buffer=xb, rcp=rcp)
            assert want[0] in (K_ASYNC, K_MOD_ASYNC)
            _assert_form(run_sparse(job, method, active, dn, x_buffer=xb, rcp=rcp), want, f"{name} {dn} {method}")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every other route to the generic kernel
# ---------------------------------------------------------------------------------------------------------------------
BASE = (256, 136, 64, 64, 24, 3)
ROUTES = {"odd_W": ((250, 136, 64, 64, 24, 3), (), 0), "odd_tile_w": ((256, 136, 62, 62, 24, 3), (), 0),
          "tiles": (BASE, ("tiles",), 0), "weights": (BASE, ("weights",), 0), "rcp": (BASE, ("rcp",), 0),
          "x_out": (BASE, ("x_out",), 0), "x_buffer": (BASE, ("x_buffer",), 0), "rescale": (BASE, ("rescale",), 0),
          "tile_weights": (BASE, ("tile_weights",), 0), "tall": ((64, 2056, 16, 16, 8, 16), (), 0),
          "force": (BASE, (), FORCE_GENERIC)}
ROUTE_METHODS = {"md": ["odd_W", "odd_tile_w", "tiles", "weights", "rcp", "x_out", "x_buffer", "tall", "force"],
                 "mod": ["odd_W", "odd_tile_w", "tiles", "rescale", "x_buffer", "tile_weights", "tall", "force"]}
ROUTE_CASES = [(m, r, dn) for m, rs in ROUTE_METHODS.items() for r in rs for dn in DTYPES]


@gpu
@pytest.mark.parametrize("method,route,dn", ROUTE_CASES, ids=[f"{m}-{r}-{dn}" for m, r, dn in ROUTE_CASES])
def test_sparse_generic_routes(method, route, dn):
    geom, shift, flags = ROUTES[route]
    job = Job(*geom, N=1, C=2)
    es = es_of(dn)
    if route == "tall":
        assert job.geo.metric("patch_rows", es) > 256 and 0 < job.geo.metric("as", es) <= AS_MAX_VISITS
    active = np.random.default_rng(11).random(job.T) < 0.5
    variants = [(True, False), (False, dn != "f32" or route == "rcp")] if method == "md" else [(True, False)]
    for xb, rcp in variants:
        if route == "x_buffer" and not xb:
            continue
        rcp = rcp or route == "rcp"
        want = expected_form(job, method, dn, x_buffer=xb, rcp=rcp, shift=shift, flags=flags)
        assert want == generic_form(method, dn, dn)
        _assert_form(run_sparse(job, method, active, dn, x_buffer=xb, rcp=rcp, shift=shift, flags=flags), want, f"{route} {xb} {rcp}")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: flags and arguments
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_one_plane_and_no_pdl_change_nothing(dn):
    job = Job(256, 256, 96, 96, 80, 8, N=2, C=2)
    active = np.random.default_rng(5).random(job.T) < 0.5
    for method in ("md", "mod"):
        rcp = method == "md" and dn != "f32"
        want = expected_form(job, method, dn, x_buffer=False, rcp=rcp)
        for flags in (0, ONE_PLANE, NO_PDL, ONE_PLANE | NO_PDL):
            _assert_form(run_sparse(job, method, active, dn, x_buffer=False, rcp=rcp, flags=flags), want, f"{method} flags={flags:#x}")


@gpu
def test_rcp_weights_are_ignored_by_an_fp32_blend():
    job = Job(256, 136, 64, 64, 24, 3, N=1, C=2)
    active = np.random.default_rng(6).random(job.T) < 0.5
    for xb in (False, True):
        traced = run_sparse(job, "md", active, "f32", x_buffer=xb, rcp=True)
        _assert_form(traced, async_form("f32", xb, False), "fp32 with rcp_weights")
        if traced is not None:
            assert all(a[2] == "false" for a in template_args(traced[1], K_ASYNC)), sorted(traced[1])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: batch tables and slot tables
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_permuted_slot_tables(dn, method):
    """Any slot table whose positions 0..K-1 each appear once, with the compact batches permuted to match, gives the monotone
    table's bits (the oracle's), on the cp.async and on the generic kernel."""
    job = Job(256, 256, 96, 96, 80, 5, N=1, C=2)
    for name, active in active_sets(job, es_of(dn), seed=2).items():
        if active.sum() < 2:
            continue
        for flags in (0, FORCE_GENERIC):
            want = expected_form(job, method, dn, x_buffer=True, flags=flags)
            _assert_form(run_sparse(job, method, active, dn, perm_seed=7, flags=flags), want, f"{name} permuted flags={flags}")


@gpu
@pytest.mark.parametrize("method", ["md", "mod"])
def test_more_than_128_compact_batches(method):
    """tile_bs 1 and several hundred kept tiles through the engine wrappers, which concatenate the compact batches."""
    eng = _eng()
    job = Job(512, 512, 32, 32, 8, 1, N=1, C=2)
    active = np.random.default_rng(8).random(job.T) < 0.7
    assert active.sum() > 128
    g, N, C = job.g, job.N, job.C
    tiles = job.tiles("f16")
    idx = torch.from_numpy(np.flatnonzero(active))
    compact = tiles.view(job.T, N, C, g.tile_h, g.tile_w)[idx].reshape(-1, C, g.tile_h, g.tile_w).cuda()
    outs = [compact[i * N:(i + 1) * N] for i in range(len(idx))]
    slot = eng.slot_table(active)
    slot_dev = torch.from_numpy(slot).cuda()
    box = {}
    if method == "md":
        w = torch.from_numpy(job.weights).cuda()
        r = torch.from_numpy(eng.exact_reciprocals(job.weights)).cuda()
        traced = _traced(lambda: box.setdefault("o", eng.blend_multidiffusion_sparse(g, outs, N, C, 1, w, torch.float16, slot_dev, slot,
                                                                                     rcp_weights=r)))
        torch.cuda.synchronize()
        assert_bit_equal(box["o"].cpu(), job.want("md", active, "f16", "f16")[0], "md > 128 batches")
        want = async_form("f16", False, True)
    else:
        twt, rs = torch.from_numpy(job.tile_weights).cuda(), torch.from_numpy(job.rescale).cuda()
        xb = _nan((N, C, g.H, g.W), torch.float16)
        traced = _traced(lambda: eng.blend_mixture_sparse(g, outs, N, C, 1, twt, rs, xb, slot_dev, slot))
        torch.cuda.synchronize()
        assert_bit_equal(xb.cpu(), job.want("mod", active, "f16", "f16"), "mod > 128 batches")
        want = mod_async_form("f16")
    _assert_form(traced, want, "> 128 compact batches")
    if traced is not None:
        assert any("cat" in n.lower() for n in traced[1] if not any(k in n for k in SPARSE_KERNELS)), sorted(traced[1])


@gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_65536_tile_plan_slots_through_fastdiv(dn):
    """A 256 x 256-tile plan: slot values up to 65535 are split into batch and row with the tile_bs magic (513 tiles per
    batch, 128 batches), on the cp.async and the generic kernel.  Tile 16 x 12, overlap 8: W = 2056 is a vector multiple and
    H = 1032 stays within the 256 patch rows of the cp.async tables."""
    job = Job(2056, 1032, 16, 12, 8, 513, N=1, C=1)
    assert (job.g.rows, job.g.cols, job.T, job.g.num_batches) == (256, 256, 65536, 128)
    full = np.ones(job.T, bool)
    sparse = full.copy()
    sparse[np.random.default_rng(3).random(job.T) < 0.25] = False
    sparse[-1] = True
    for name, active in (("all", full), ("75%", sparse)):
        for method in ("md", "mod"):
            for flags in (0, FORCE_GENERIC):
                want = expected_form(job, method, dn, x_buffer=True, flags=flags)
                _assert_form(run_sparse(job, method, active, dn, flags=flags, tile_bs=513), want, f"65536 tiles {name} {method} {flags}")
    _assert_form(run_sparse(job, "md", sparse, dn, perm_seed=1, tile_bs=513), expected_form(job, "md", dn), "65536 tiles permuted")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: td_grid_active_tiles at its edges
# ---------------------------------------------------------------------------------------------------------------------
def _edge_values(dt):
    one = torch.tensor(1.0, dtype=dt)
    finfo = torch.finfo(dt)
    return {"1+ulp": torch.nextafter(one, torch.tensor(2.0, dtype=dt)).item(),
            "1-ulp": torch.nextafter(one, torch.tensor(0.0, dtype=dt)).item(),
            "-0": -0.0, "+inf": float("inf"), "-inf": float("-inf"), "min_subnormal": finfo.smallest_normal * finfo.eps,
            "nan": float("nan"), "just_below_one_f16": JUST_BELOW_ONE}


@gpu
@pytest.mark.parametrize("planes", [1, 4, 8])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_active_tiles_edges(dn, planes):
    eng = _eng()
    dt = DTYPES[dn]
    g = eng.make_grid(512, 512, 96, 96, 48, 8)
    bbs = [tuple(int(v) for v in r) for r in eng.grid_bboxes_xywh(g)]
    T = len(bbs)
    for name, val in _edge_values(dt).items():
        stored = torch.tensor(val, dtype=dt)
        assert name == "just_below_one_f16" or stored.item() != 1.0 or torch.isnan(stored), name
        if name == "min_subnormal":
            assert 0 < stored.item() < torch.finfo(dt).smallest_normal
        for t in (0, T // 2 + 3, T - 1):
            x, y, w, h = bbs[t]
            for where, (pl, py, px) in (("first", (0, y, x)), ("last", (planes - 1, y + h - 1, x + w - 1))):
                m = torch.ones((planes, 512, 512), dtype=dt)
                m[pl, py, px] = val
                shaped = m[0] if planes == 1 else (m.view(2, 4, 512, 512) if planes == 8 else m)    # [h, w], [C, h, w], [N, C, h, w]
                got = eng.active_tiles(g, shaped.cuda())
                want = rule(m, bbs)
                assert np.array_equal(got, want), f"{dn} planes={planes} {name} tile {t} {where}: {np.flatnonzero(got != want)}"
                assert want[t] == (stored.item() != 1.0 or bool(torch.isnan(stored)))


@gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_active_tiles_on_a_65536_tile_grid(dn):
    eng = _eng()
    g = eng.make_grid(1028, 1028, 8, 8, 4, 64)
    assert g.num_tiles == 65536
    bbs = [tuple(int(v) for v in r) for r in eng.grid_bboxes_xywh(g)]
    m = torch.ones((4, 1028, 1028), dtype=DTYPES[dn])
    m[3, 1027, 1027] = 0.5                                  # the last element of the last plane of the last tile
    m[0, 0, 0] = float("nan")
    rng = np.random.default_rng(0)
    for _ in range(40):
        m[int(rng.integers(0, 4)), int(rng.integers(0, 1028)), int(rng.integers(0, 1028))] = -0.0
    got = eng.active_tiles(g, m.cuda())
    want = rule(m, bbs)
    assert want[0] and want[-1] and 0 < want.sum() < 65536
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: SpotDiffusion step plans
# ---------------------------------------------------------------------------------------------------------------------
K_WRAP_SC_VEC, K_WRAP_VEC, K_WRAP_GEN = "wrap_scatter_vec_kernel", "wrap_blend_vec_kernel", "wrap_blend_generic_kernel"
STEP_KERNELS = (K_ASYNC, K_VEC, K_GENERIC, K_SCATTER_ROWS, K_SCATTER_VEC, K_SCATTER_GENERIC, K_WRAP_SC_VEC, K_WRAP_VEC, K_WRAP_GEN)


def _step_forms(sg, dn, tile_dn):
    """(scatter form, blend form) the host checks choose on step plan `sg`: the bounded kernels of td_diffusion.cu, or the
    vector kernels of td_wrap.cu on a periodic plan (W and tile_w are vector multiples in every geometry here)."""
    es = es_of(dn)
    if sg.g.wrap:
        vec = 16 // es
        assert sg.W % vec == 0 and sg.tw % vec == 0
        sc = (K_WRAP_SC_VEC, ("float" if dn == "f32" else "__half",))
        if tile_dn != dn:
            return sc, (K_WRAP_GEN, (CT[tile_dn], CT[dn], "0"))
        return sc, (K_WRAP_VEC, (CT[dn], "0", "false", "false"))
    sc = sg.expected("scatter", es, 0)
    if tile_dn != dn:
        return sc, K_GENERIC
    return sc, sg.expected("md", es, 0)


def _forms_only(traced):
    """(forms, names) of a traced step-plan call: bounded kernels by name, td_wrap.cu kernels with their template arguments."""
    if traced is None:
        return None
    names = traced[1]
    wrapped = {(k, tuple(a)) for k in (K_WRAP_SC_VEC, K_WRAP_VEC, K_WRAP_GEN) for a in template_args(names, k)}
    return forms(names) | wrapped, names


def run_step(W, H, t, ov, wrap, sx, sy, dn, tile_dn=None, bs=8, N=1, C=4):
    """Scatter, fake UNet on the CPU, blend with the device count canvas (and reciprocals when they apply) on one step plan;
    bit-checked against spot_oracle.  Returns the traced scatter and blend and the step plan."""
    eng = _eng()
    tile_dn = tile_dn or dn
    sg = SpotGeo(eng, W, H, t, t, ov, bs, wrap, sx, sy)
    plan, g = sg.plan, sg.g
    x = synth.latent(W + 3 * H + sx, (N, C, H, W), DTYPES[dn])
    xd = x.cuda()
    box = {}
    sc = _traced(lambda: box.setdefault("tiles", eng.scatter_tiles(g, xd)), STEP_KERNELS)
    torch.cuda.synchronize()
    want_tiles = wo.scatter(x, plan.bboxes) if wrap else blend.scatter_tiles(x, plan.bboxes)
    assert_bit_equal(box["tiles"].cpu(), want_tiles, f"scatter {W}x{H} {t}/{ov} wrap={wrap} ({sx},{sy}) {dn}")
    den = lambda tl, bb: synth.fake_denoise(tl, bb, N).to(DTYPES[tile_dn])        # noqa: E731
    want = so.step(x, plan, den)
    outs = [den(want_tiles[i * plan.tile_bs * N:(i * plan.tile_bs + len(bb)) * N], bb).cuda() for i, bb in enumerate(plan.batched_bboxes)]
    w = torch.empty(H * W, device="cuda")
    fast = eng.counts_allow_fast_divide(g)
    r = torch.empty(H * W, device="cuda") if fast else None
    eng.grid_counts(g, w, r)
    bl = _traced(lambda: box.__setitem__("out", eng.blend_multidiffusion(g, outs, N, C, g.tile_bs, w, DTYPES[dn], rcp_weights=r)), STEP_KERNELS)
    torch.cuda.synchronize()
    assert_bit_equal(box["out"].cpu(), want, f"blend {W}x{H} {t}/{ov} wrap={wrap} ({sx},{sy}) {dn} tile={tile_dn} fast={fast}")
    return _forms_only(sc), _forms_only(bl), sg


STEP_CASES = [(geom, dn) for geom in SPOT_GEOMS for dn in DTYPES]


@gpu
@pytest.mark.parametrize("geom,dn", STEP_CASES, ids=[f"{g[0]}x{g[1]}_{g[2]}_{g[3]}_w{g[4]}-{dn}" for g, dn in STEP_CASES])
def test_step_plans_at_ui_sizes(geom, dn):
    W, H, t, ov, wrap = geom
    for sx, sy in _shifts(W, H, t, t, ov, wrap):
        sc, bl, sg = run_step(W, H, t, ov, wrap, sx, sy, dn)
        want_sc, want_bl = _step_forms(sg, dn, dn)
        if sc is not None:
            assert sc[0] == {want_sc}, (geom, dn, (sx, sy), sorted(sc[1]))
            assert bl[0] == {want_bl}, (geom, dn, (sx, sy), sorted(bl[1]))
        if geom in CROSSING and t == 128 and dn != "f32":
            assert want_bl == K_VEC, "a 128 / 112 step plan is past the cp.async limit"


@gpu
def test_base_plan_and_step_plans_of_128_112_take_different_forms():
    """In fp16 the 128 / 112 base plan runs blend_md_async_kernel and its step plans blend_grid_vec_kernel."""
    W, H, t, ov = 256, 256, 128, 112
    geo = Geo(_eng(), W, H, t, t, ov, 8)
    assert geo.expected("md", 2, 0) == K_ASYNC
    plan = tiling.GridPlan(W, H, t, t, ov, 8, False)
    x = synth.latent(1, (1, 4, H, W), torch.float16)
    den = lambda tl, bb: synth.fake_denoise(tl, bb, 1)            # noqa: E731
    want = blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, den)
    outs = [den(blend.scatter_tiles(x, bb), bb).cuda() for bb in plan.batched_bboxes]
    w = torch.from_numpy(plan.weights).cuda()
    r = torch.from_numpy(_eng().exact_reciprocals(plan.weights)).cuda()
    box = {}
    bl = _forms_only(_traced(lambda: box.__setitem__("o", _eng().blend_multidiffusion(geo.g, outs, 1, 4, geo.g.tile_bs, w, torch.float16,
                                                                                       rcp_weights=r)), STEP_KERNELS))
    torch.cuda.synchronize()
    assert_bit_equal(box["o"].cpu(), want, "128 / 112 base plan")
    if bl is not None:
        assert bl[0] == {K_ASYNC}, sorted(bl[1])
    for sx, sy in _shifts(W, H, t, t, ov, 0):
        _, bl, sg = run_step(W, H, t, ov, 0, sx, sy, "f16")
        assert sg.metric("as", 2) > AS_MAX_VISITS
        if bl is not None:
            assert bl[0] == {K_VEC}, sorted(bl[1])


@gpu
@pytest.mark.parametrize("geom", [CFG2[1], PANORAMA[1], (256, 256, 128, 112, 0)], ids=["cfg2", "panorama_wrapx", "128_112"])
def test_step_plan_fp32_tiles_on_an_fp16_latent(geom):
    """The UNet's fp32 output on an fp16 latent takes the generic kernel on a step plan."""
    W, H, t, ov, wrap = geom
    lo_x, hi_x, lo_y, hi_y = so.bounds(W, H, t, t, ov, wrap)
    sx, sy = (lo_x + hi_x) // 2, hi_y - 1
    sc, bl, sg = run_step(W, H, t, ov, wrap, sx, sy, "f16", tile_dn="f32")
    want_sc, want_bl = _step_forms(sg, "f16", "f32")
    if bl is not None:
        assert sc[0] == {want_sc} and bl[0] == {want_bl}, (sorted(sc[1]), sorted(bl[1]))
        if not wrap:
            assert template_args(bl[1], K_GENERIC) == [["float", "__half", "0", "false"]], sorted(bl[1])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the SpotDiffusion delegate where its step plans leave the cp.async limit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def shared():
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
    model = types.SimpleNamespace(cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="concat"))
    host.use_shared(types.SimpleNamespace(state=state, sd_model=model))
    host._a1111_cache.clear()
    yield state
    host.use_shared(None)


@gpu
def test_delegate_three_calls_at_128_112(shared):
    """Three consecutive k-diffusion calls of the SpotDiffusion delegate on a 256^2 fp16 latent, tile 128 / overlap 112,
    against spot_oracle: each call's step plan holds 81 visits per patch."""
    from multidiffusion_upscaler_for_automatic1111_b200 import SpotDiffusion
    W, H, t, ov, bs, N, C, seed = 256, 256, 128, 112, 8, 1, 4, 5

    def unet(x_tile, ts, cond):
        return (wo.blur_denoise(x_tile).float() + cond["c_concat"][0].float()).to(x_tile.dtype)
    sampler = type("KDiffusionSampler", (), {})()
    sampler.model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=unet), image_cfg_scale=None, step=0)
    d = SpotDiffusion(types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True), sampler)
    d.init_grid_bbox(t, t, ov, bs, shift_seed=seed)
    d.init_done()
    d.hook()
    gen = torch.Generator().manual_seed(2)
    x = (torch.randn((N, C, H, W), generator=gen) * 2).half()
    icond = torch.randn((N, C, H, W), generator=gen).half()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4).cuda()], "c_concat": [icond.cuda()]}
    denoise = lambda xt, bb: (wo.blur_denoise(xt).float() + wo.scatter(icond, bb).float()).to(xt.dtype)   # noqa: E731
    for k, (sx, sy) in enumerate(so.schedule(seed, so.bounds(W, H, t, t, ov, 0), 3)):
        got = d.sampler.model_wrap_cfg.inner_model.forward(x.cuda(), torch.ones(N).cuda(), cond=cond)
        plan = so.SpotPlan(W, H, t, t, ov, bs, 0, sx, sy)
        assert [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb] == plan.bboxes, f"call {k}"
        assert SpotGeo(_eng(), W, H, t, t, ov, bs, 0, sx, sy).metric("as", 2) > AS_MAX_VISITS
        assert_bit_equal(got.cpu(), so.step(x, plan, denoise), f"call {k} ({sx}, {sy})")
        x = got.cpu().half()
