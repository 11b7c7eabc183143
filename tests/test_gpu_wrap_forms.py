"""Seamless tiling (csrc/td_wrap.cu) at every kernel form, dtype pair and limit, bit for bit against tests/wrap_oracle.py.

Every MultiDiffusion / Mixture of Diffusers step on a plan with a wrap bit runs through td_wrap.cu.  Its scatter and
blends have a vector form (16-byte loads, a funnel shift across the seam, a two-range origin search) and a generic form
(one element per thread, any width / alignment, tile and canvas dtypes independent).  The entries take the generic form
when any of these holds: W % VEC, tile_w % VEC, a 16-byte misaligned buffer, a tile dtype other than the canvas dtype,
TD_FLAG_FORCE_GENERIC.  Here each condition is broken on its own; every template instantiation that can launch is run
and named (`FORM_MATRIX`); the plans reach 256 origins per axis, the 32767 canvas, N*C = 65535 planes, 128 batch
tensors, 36 visits per pixel, tiles as wide and as tall as the canvas, origins far from the search estimate and
one-vector canvases.  The CPU part pins the oracle's mixed-dtype rounding, shows that each bit check catches an injected
kernel defect, and that every grid entry refuses origins out of order.
"""
import ctypes
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal
from test_gpu_blend_limits import launched, template_args

WRAP_XY = wo.WRAP_X | wo.WRAP_Y
WRAPS = [wo.WRAP_X, wo.WRAP_Y, WRAP_XY]
FORCE_GENERIC = 1

# ---------------------------------------------------------------------------------------------------------------------
# which template ran
# ---------------------------------------------------------------------------------------------------------------------
K_SC_VEC, K_SC_GEN = "wrap_scatter_vec_kernel", "wrap_scatter_generic_kernel"
K_VEC, K_GEN = "wrap_blend_vec_kernel", "wrap_blend_generic_kernel"
KERNELS = (K_SC_VEC, K_SC_GEN, K_VEC, K_GEN)
CT = {"f16": "__half", "bf16": "__nv_bfloat16", "f32": "float"}   # template argument spelling of each dtype
MODE = {"md": "0", "mod": "1"}
H_, B_, F_ = "__half", "__nv_bfloat16", "float"

# Every instantiation of td_wrap.cu that an entry can launch.  The scatter moves fp16 and bf16 as opaque 16-bit words
# (<__half>).  Vector blends: <T, MODE, WRITE_BUF, WINDOW>; WRITE_BUF is set when MultiDiffusion gets an x_buffer and
# always for Mixture of Diffusers (its result is the buffer), so <T, 1, false, *> is compiled but unreachable; WINDOW is
# the row-window form of td_blend_*_wrap_rows.  Generic blends: <TIn, TAcc, MODE> for all nine dtype pairs.
FORM_MATRIX = [
    (K_SC_VEC, (H_,)), (K_SC_VEC, (F_,)), (K_SC_GEN, (H_,)), (K_SC_GEN, (F_,)),
    (K_VEC, (H_, "0", "false", "false")), (K_VEC, (H_, "0", "true", "false")),
    (K_VEC, (H_, "0", "false", "true")), (K_VEC, (H_, "0", "true", "true")),
    (K_VEC, (B_, "0", "false", "false")), (K_VEC, (B_, "0", "true", "false")),
    (K_VEC, (B_, "0", "false", "true")), (K_VEC, (B_, "0", "true", "true")),
    (K_VEC, (F_, "0", "false", "false")), (K_VEC, (F_, "0", "true", "false")),
    (K_VEC, (F_, "0", "false", "true")), (K_VEC, (F_, "0", "true", "true")),
    (K_VEC, (H_, "1", "true", "false")), (K_VEC, (H_, "1", "true", "true")),
    (K_VEC, (B_, "1", "true", "false")), (K_VEC, (B_, "1", "true", "true")),
    (K_VEC, (F_, "1", "true", "false")), (K_VEC, (F_, "1", "true", "true")),
    (K_GEN, (H_, H_, "0")), (K_GEN, (H_, B_, "0")), (K_GEN, (H_, F_, "0")),
    (K_GEN, (B_, H_, "0")), (K_GEN, (B_, B_, "0")), (K_GEN, (B_, F_, "0")),
    (K_GEN, (F_, H_, "0")), (K_GEN, (F_, B_, "0")), (K_GEN, (F_, F_, "0")),
    (K_GEN, (H_, H_, "1")), (K_GEN, (H_, B_, "1")), (K_GEN, (H_, F_, "1")),
    (K_GEN, (B_, H_, "1")), (K_GEN, (B_, B_, "1")), (K_GEN, (B_, F_, "1")),
    (K_GEN, (F_, H_, "1")), (K_GEN, (F_, B_, "1")), (K_GEN, (F_, F_, "1")),
]


def vec_form(op, dn, buf=True, window=False):
    if op == "scatter":
        return (K_SC_VEC, (F_ if dn == "f32" else H_,))
    return (K_VEC, (CT[dn], MODE[op], "true" if buf or op == "mod" else "false", "true" if window else "false"))


def generic_form(op, dn, tile_dn=None):
    if op == "scatter":
        return (K_SC_GEN, (F_ if dn == "f32" else H_,))
    return (K_GEN, (CT[tile_dn or dn], CT[dn], MODE[op]))


# Which kernel ran is read from a CUPTI trace, and that trace is reliable only in a young process (late in a long GPU
# session most profiler sessions come back without kernel records).  So the form assertions run in a fresh interpreter
# (`test_launched_forms_in_a_fresh_process`), and in this process `_forms` only runs the call; every bit check runs in both.
FORMS_CHILD = os.environ.get("TD_WRAP_FORMS_CHILD") == "1"


class _NotTraced:
    """What `_forms` returns outside the child interpreter: equal to any expected form set (the child asserts it)."""

    def __eq__(self, other):
        return True

    __hash__ = None

    def __repr__(self):
        return "<forms asserted in the child interpreter>"


def _forms(fn):
    """{(kernel, template arguments)} of the td_wrap.cu kernels `fn` launched (in the child interpreter; see above)."""
    if not FORMS_CHILD:
        fn()
        return _NotTraced()
    names = launched(fn)
    return {(k, tuple(a)) for k in KERNELS for a in template_args(names, k)}


FORM_TESTS = "not mixed_tile_and_canvas and not fresh_process"


@pytest.mark.gpu
def test_launched_forms_in_a_fresh_process():
    """The tests that assert which template ran, rerun in a fresh interpreter where the kernel trace is complete."""
    if FORMS_CHILD:
        pytest.skip("already the child interpreter")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    cmd = [sys.executable, *flags, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k", FORM_TESTS]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(cmd, cwd=root, env=dict(os.environ, TD_WRAP_FORMS_CHILD="1"), capture_output=True, text=True, timeout=1200)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail


# ---------------------------------------------------------------------------------------------------------------------
# plans, inputs and one call of each entry, checked bit for bit
# ---------------------------------------------------------------------------------------------------------------------
class Case:
    """A periodic plan -- from td_grid_init (`ov` given) or with hand-made origins (`xs`, `ys`) -- and the oracle's inputs."""

    def __init__(self, W, H, tw, th, wrap, ov=None, bs=4, xs=None, ys=None, N=2, C=3):
        from multidiffusion_upscaler_for_automatic1111_b200 import engine
        from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
        from oracle import tiling
        self.N, self.C = N, C
        if xs is None:
            self.g = g = engine.make_grid(W, H, tw, th, ov, bs, wrap=wrap)
            plan = wo.WrapPlan(W, H, tw, th, ov, bs, wrap)
            assert (list(g.xs[:g.cols]), list(g.ys[:g.rows])) == (plan.xs, plan.ys), "engine plan differs from the oracle's"
            assert (g.num_batches, g.tile_bs) == (plan.num_batches, plan.tile_bs)
            self.bboxes = plan.bboxes
        else:
            self.g = g = TdGrid()
            g.W, g.H, g.tile_w, g.tile_h, g.overlap, g.wrap = W, H, tw, th, 0, wrap
            g.rows, g.cols, g.num_tiles = len(ys), len(xs), len(ys) * len(xs)
            g.num_batches = -(-g.num_tiles // bs)
            g.tile_bs = bs
            for i, v in enumerate(xs):
                g.xs[i] = v
            for i, v in enumerate(ys):
                g.ys[i] = v
            self.bboxes = [(x, y, tw, th) for y in ys for x in xs]
        self.W, self.H, self.tw, self.th, self.tile_bs = g.W, g.H, g.tile_w, g.tile_h, g.tile_bs
        self.T = g.num_tiles
        self.batched = [self.bboxes[i:i + self.tile_bs] for i in range(0, self.T, self.tile_bs)]
        self.shape = (N, C, self.H, self.W)
        self.weights = wo.weights(self.bboxes, self.W, self.H)
        self.tile_weights = tiling.gaussian_weights(self.tw, self.th)
        with np.errstate(divide="ignore"):
            self.rescale = (np.float32(1.0) / wo.weights(self.bboxes, self.W, self.H, self.tile_weights)).astype(np.float32)

    @functools.lru_cache(maxsize=None)
    def x(self, dn):
        return (torch.randn(self.shape, generator=torch.Generator().manual_seed(self.W + 7 * self.H)) * 2).to(DTYPES[dn])

    @functools.lru_cache(maxsize=None)
    def outs(self, dn):
        gen = torch.Generator().manual_seed(3 * self.W + self.H)
        return [(torch.randn((len(b) * self.N, self.C, self.th, self.tw), generator=gen) * 1.5).to(DTYPES[dn]) for b in self.batched]

    @functools.lru_cache(maxsize=None)
    def want(self, op, dn, tile_dn):
        """The oracle's result: (fp32 output, canvas-dtype accumulator) for MultiDiffusion, the accumulator for MoD."""
        outs = self.outs(tile_dn)
        if op == "md":
            return wo.blend_md(outs, self.batched, self.N, self.shape, DTYPES[dn], self.weights)
        return wo.blend_mod(outs, self.batched, self.N, self.shape, DTYPES[dn], self.tile_weights, self.rescale)


@functools.lru_cache(maxsize=None)
def case(*args, **kw):
    return Case(*args, **kw)


def _shifted(t):
    """A copy of `t` whose data pointer is one element past a 16-byte boundary (an offset view into a larger buffer)."""
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def _nan(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def run_scatter(c, dn, flags=0, shift=(), rng=None):
    """One scatter of case `c` (tiles [rng)), checked against the oracle; returns the forms it launched."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    b, e = rng if rng is not None else (0, c.T)
    x = c.x(dn)
    xd = x.cuda()
    if "x" in shift:
        xd = _shifted(xd)
    out = _nan(((e - b) * c.N, c.C, c.th, c.tw), x.dtype)
    if "tiles" in shift:
        out = _shifted(out)
    forms = _forms(lambda: engine.scatter_tiles(c.g, xd, out=out, tile_begin=b, tile_end=e, flags=flags))
    assert_bit_equal(out.cpu(), wo.scatter(x, c.bboxes[b:e]), f"scatter {dn} {c.shape} [{b},{e}) flags={flags} shift={shift}")
    return forms


def run_blend(c, op, dn, tile_dn=None, x_buffer=True, flags=0, shift=()):
    """One td_blend_multidiffusion / td_blend_mixture of case `c`, checked bit for bit; returns the forms it launched.
    `shift` names the buffers passed one element off 16-byte alignment; `tile_dn` the tile dtype (default: the canvas')."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    tile_dn = tile_dn or dn
    N, C, acc = c.N, c.C, DTYPES[dn]
    douts = [o.cuda() for o in c.outs(tile_dn)]
    if "tiles" in shift:
        douts[-1] = _shifted(douts[-1])
    tag = f"{op} {dn} tile={tile_dn} {c.shape} xs={list(c.g.xs[:c.g.cols])} flags={flags} x_buffer={x_buffer} shift={shift}"
    if op == "md":
        want, want_buf = c.want("md", dn, tile_dn)
        w = torch.from_numpy(c.weights).cuda()
        if "weights" in shift:
            w = _shifted(w)
        r = None
        if "rcp_weights" in shift:
            r = _shifted(torch.from_numpy(engine.exact_reciprocals(c.weights)).cuda())
        out = _nan(c.shape, torch.float32)
        if "x_out" in shift:
            out = _shifted(out)
        xb = _nan(c.shape, acc) if x_buffer else None
        if xb is not None and "x_buffer" in shift:
            xb = _shifted(xb)
        forms = _forms(lambda: engine.blend_multidiffusion(c.g, douts, N, C, c.tile_bs, w, acc, x_buffer=xb, flags=flags, out=out,
                                                           rcp_weights=r))
        assert_bit_equal(out.cpu(), want, tag)
        if xb is not None:
            assert_bit_equal(xb.cpu(), want_buf, tag + " x_buffer")
        return forms
    assert np.isfinite(c.rescale).all(), "an infinite rescale makes 0 * inf: NaN payloads differ between CPU and GPU"
    want = c.want("mod", dn, tile_dn)
    tw = torch.from_numpy(c.tile_weights).cuda()
    if "tile_weights" in shift:
        tw = _shifted(tw)
    rs = torch.from_numpy(c.rescale).cuda()
    if "rescale" in shift:
        rs = _shifted(rs)
    xb = _nan(c.shape, acc)
    if "x_buffer" in shift:
        xb = _shifted(xb)
    forms = _forms(lambda: engine.blend_mixture(c.g, douts, N, C, c.tile_bs, tw, rs, xb, flags=flags))
    assert_bit_equal(xb.cpu(), want, tag)
    return forms


def run_rows(c, op, dn, windows, x_buffer=True):
    """td_blend_*_wrap_rows over row windows that together cover the canvas (no halo wait), checked bit for bit."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N, C, acc = c.N, c.C, DTYPES[dn]
    tiles = torch.cat(c.outs(dn)).cuda()                       # tile-major: tile row i is one contiguous band
    band = c.g.cols * N * C * c.th * c.tw * tiles.element_size()
    ptrs = [tiles.data_ptr() + i * band for i in range(c.g.rows)]
    tag = f"{op} rows {dn} {c.shape} windows={windows} x_buffer={x_buffer}"
    if op == "md":
        want, want_buf = c.want("md", dn, dn)
        w = torch.from_numpy(c.weights).cuda()
        out = _nan(c.shape, torch.float32)
        xb = _nan(c.shape, acc) if x_buffer else None
        forms = _forms(lambda: [engine.blend_multidiffusion_wrap_rows(c.g, ptrs, N, C, acc, w, out, lo, hi, x_buffer=xb) for lo, hi in windows])
        assert_bit_equal(out.cpu(), want, tag)
        if xb is not None:
            assert_bit_equal(xb.cpu(), want_buf, tag + " x_buffer")
        return forms
    tw = torch.from_numpy(c.tile_weights).cuda()
    rs = torch.from_numpy(c.rescale).cuda()
    xb = _nan(c.shape, acc)
    forms = _forms(lambda: [engine.blend_mixture_wrap_rows(c.g, ptrs, N, C, acc, tw, rs, xb, lo, hi) for lo, hi in windows])
    assert_bit_equal(xb.cpu(), c.want("mod", dn, dn), tag)
    return forms


def run_all(c, dn, flags=0, expect=None):
    """Scatter, MultiDiffusion with and without x_buffer, Mixture of Diffusers; each must run form `expect(op, buf)`."""
    got = run_scatter(c, dn, flags)
    assert got == {expect("scatter", True)}, got
    for op, buf in (("md", True), ("md", False), ("mod", True)):
        got = run_blend(c, op, dn, x_buffer=buf, flags=flags)
        assert got == {expect(op, buf)}, (op, buf, got)


def vector(dn):
    return lambda op, buf: vec_form(op, dn, buf)


def generic(dn):
    return lambda op, buf: generic_form(op, dn)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the form matrix: each vector condition broken on its own
# ---------------------------------------------------------------------------------------------------------------------
BASE = (120, 64, 40, 24, WRAP_XY)        # periodic origins 0, 30, 60, 90: unaligned windows, some crossing the seam
ODD_W = (118, 64, 40, 24, WRAP_XY)       # W % VEC != 0 for every dtype (origins 0, 29, 59, 88)
ODD_TW = (120, 64, 42, 24, WRAP_XY)      # tile_w % VEC != 0 for every dtype
OTHER = {"f16": "f32", "bf16": "f16", "f32": "bf16"}

# condition -> (geometry, misaligned buffers, flags, mixed tile dtype); "none" is the aligned control, "tile_weights"
# is not a condition (MoD reads the tile weights one float at a time): the vector form must stay
CONDITIONS = {
    "none": (BASE, (), 0, False), "W": (ODD_W, (), 0, False), "tw": (ODD_TW, (), 0, False), "force": (BASE, (), FORCE_GENERIC, False),
    "x": (BASE, ("x",), 0, False), "tiles": (BASE, ("tiles",), 0, False), "weights": (BASE, ("weights",), 0, False),
    "rcp_weights": (BASE, ("rcp_weights",), 0, False), "x_out": (BASE, ("x_out",), 0, False),
    "x_buffer": (BASE, ("x_buffer",), 0, False), "rescale": (BASE, ("rescale",), 0, False),
    "tile_weights": (BASE, ("tile_weights",), 0, False), "mixed": (BASE, (), 0, True),
}
OP_CONDITIONS = {"scatter": ["none", "W", "tw", "x", "tiles", "force"],
                 "md": ["none", "W", "tw", "tiles", "weights", "rcp_weights", "x_out", "x_buffer", "mixed", "force"],
                 "mod": ["none", "W", "tw", "tiles", "rescale", "x_buffer", "mixed", "force", "tile_weights"]}
COND_CASES = [(op, cond, dn) for op, conds in OP_CONDITIONS.items() for cond in conds for dn in DTYPES]


@pytest.mark.gpu
@pytest.mark.parametrize("op,cond,dn", COND_CASES, ids=[f"{op}-{cond}-{dn}" for op, cond, dn in COND_CASES])
def test_each_vector_condition_falls_back_to_generic(op, cond, dn):
    geom, shift, flags, mixed = CONDITIONS[cond]
    c = case(*geom, ov=8)
    tile_dn = OTHER[dn] if mixed else dn
    keeps_vector = cond in ("none", "tile_weights")
    want = vec_form(op, dn) if keeps_vector else generic_form(op, dn, tile_dn)
    if op == "scatter":
        got = run_scatter(c, dn, flags, shift)
    else:
        got = run_blend(c, op, dn, tile_dn=tile_dn, flags=flags, shift=shift)
    assert got == {want}, f"{op} {cond} {dn}: ran {got}"


WINDOW_CASES = [((120, 64, 40, 24, WRAP_XY), [(0, 24), (24, 64)]),
                ((120, 37, 40, 20, WRAP_XY), [(16, 37), (0, 16)]),      # a partial last CTA row; windows out of order
                ((64, 48, 16, 16, wo.WRAP_Y), [(0, 8), (8, 48)])]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("op,buf", [("md", True), ("md", False), ("mod", True)])
@pytest.mark.parametrize("k", range(len(WINDOW_CASES)))
def test_window_forms(k, op, buf, dn):
    """td_blend_*_wrap_rows without a halo wait: the WINDOW = true instantiations, row window by row window."""
    (W, H, tw, th, wrap), windows = WINDOW_CASES[k]
    c = case(W, H, tw, th, wrap, ov=8)
    got = run_rows(c, op, dn, windows, x_buffer=buf)
    assert got == {vec_form(op, dn, buf, window=True)}, got


@pytest.mark.gpu
def test_every_instantiation_launches():
    """Each entry of FORM_MATRIX launches on some call, and nothing outside it does."""
    c = case(*BASE, ov=8)
    seen = set()

    def add(forms):
        if FORMS_CHILD:
            seen.update(forms)

    for dn in DTYPES:
        add(run_scatter(c, dn))
        add(run_scatter(c, dn, FORCE_GENERIC))
        for buf in (True, False):
            add(run_blend(c, "md", dn, x_buffer=buf))
            add(run_rows(c, "md", dn, [(0, 32), (32, 64)], x_buffer=buf))
        add(run_blend(c, "mod", dn))
        add(run_rows(c, "mod", dn, [(0, 32), (32, 64)]))
        for tile_dn in DTYPES:
            add(run_blend(c, "md", dn, tile_dn=tile_dn, flags=FORCE_GENERIC))
            add(run_blend(c, "mod", dn, tile_dn=tile_dn, flags=FORCE_GENERIC))
    if FORMS_CHILD:
        assert len(set(FORM_MATRIX)) == len(FORM_MATRIX) == 40
        assert seen == set(FORM_MATRIX), f"missing {sorted(set(FORM_MATRIX) - seen)}, unlisted {sorted(seen - set(FORM_MATRIX))}"


# ---------------------------------------------------------------------------------------------------------------------
# 2. tile dtype != canvas dtype (the UNet's output dtype differs from the latent's)
# ---------------------------------------------------------------------------------------------------------------------
MIXED = [(t, a) for t in DTYPES for a in DTYPES if t != a]   # (tile, canvas)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_dn,dn", MIXED)
@pytest.mark.parametrize("wrap", WRAPS)
@pytest.mark.parametrize("geom", [(120, 64, 40, 24, 8, 4), (100, 37, 33, 20, 8, 3)], ids=["seam_windows", "odd_width"])
def test_mixed_tile_and_canvas_dtypes(geom, wrap, tile_dn, dn):
    """`x_buffer += tile` rounds round_TAcc(float(acc) + float(tile)); MoD adds tile * (tile_weights * rescale) in fp32."""
    W, H, tw, th, ov, bs = geom
    c = case(W, H, tw, th, wrap, ov=ov, bs=bs)
    for buf in (True, False):
        run_blend(c, "md", dn, tile_dn=tile_dn, x_buffer=buf)
    run_blend(c, "mod", dn, tile_dn=tile_dn)


def test_wrap_oracle_at_wrap_zero_is_the_bounded_oracle_for_mixed_dtypes():
    """At wrap = 0, tests/wrap_oracle.py equals oracle/blend.py for every unequal (tile, canvas) pair, and both equal the
    explicit rounding the kernels implement: acc = round_TAcc(float(acc) + float(tile)) per add, and for MoD
    round_TAcc(float(acc) + float(tile) * (tile_weights * rescale)) with an fp32 product."""
    from oracle import blend, tiling
    W, H, tw, th, ov, bs, N, C = 64, 48, 16, 16, 8, 4, 2, 3
    for tile_dn, dn in MIXED:
        plan = wo.WrapPlan(W, H, tw, th, ov, bs, 0, gaussian=True)
        gp = tiling.GridPlan(W, H, tw, th, ov, bs, True)
        assert plan.bboxes == [tuple(b) for b in gp.bboxes]
        gen = torch.Generator().manual_seed(5)
        outs = [(torch.randn((len(b) * N, C, th, tw), generator=gen) * 1.5).to(DTYPES[tile_dn]) for b in plan.batched_bboxes]
        acc = DTYPES[dn]
        weights = wo.weights(plan.bboxes, W, H)
        twt, rs = torch.from_numpy(plan.tile_weights), torch.from_numpy(plan.rescale_factor).view(1, 1, H, W)
        got_md, got_buf = wo.blend_md(outs, plan.batched_bboxes, N, (N, C, H, W), acc, weights)
        got_mod = wo.blend_mod(outs, plan.batched_bboxes, N, (N, C, H, W), acc, plan.tile_weights, plan.rescale_factor)
        ref_buf, ref_mod = torch.zeros((N, C, H, W), dtype=acc), torch.zeros((N, C, H, W), dtype=acc)
        exp_buf, exp_mod = ref_buf.clone(), ref_mod.clone()
        for out, bbs in zip(outs, plan.batched_bboxes):
            blend.accumulate_md(ref_buf, out, bbs, N)
            blend.accumulate_mod(ref_mod, out, bbs, N, twt, rs)
            for i, (x, y, w, h) in enumerate(bbs):
                sl = (slice(None), slice(None), slice(y, y + h), slice(x, x + w))
                t = out[i * N:(i + 1) * N].float()
                exp_buf[sl] = (exp_buf[sl].float() + t).to(acc)
                exp_mod[sl] = (exp_mod[sl].float() + t * (twt * rs[sl])).to(acc)
        w4 = torch.from_numpy(weights).view(1, 1, H, W)
        tag = f"tile={tile_dn} canvas={dn}"
        assert_bit_equal(got_buf, ref_buf, tag + " MD buffer vs oracle/blend.py")
        assert_bit_equal(got_buf, exp_buf, tag + " MD buffer vs the explicit rounding")
        assert_bit_equal(got_md, blend.normalise_md(ref_buf, w4).float(), tag + " MD output")
        assert_bit_equal(got_mod, ref_mod, tag + " MoD vs oracle/blend.py")
        assert_bit_equal(got_mod, exp_mod, tag + " MoD vs the explicit rounding")


# ---------------------------------------------------------------------------------------------------------------------
# 3. limits, each at the limit and one past it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("axis", ["x", "y"])
def test_256_periodic_origins_on_the_widest_canvas(axis):
    """W = 32760, tile 192, overlap 64: stride 128, exactly 256 origins (TD_MAX_GRID_DIM) and a vector path in fp16.  The
    other tile argument is at least 68: td_grid_init clamps the overlap to min(unclamped tile args) - 4.  (The y case is
    128 wide: the gaussian tile weights of a tall 8-wide tile underflow to 0.)  257 origins are refused by td_grid_init."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_UNSUPPORTED, TdError
    L = 32760
    geom = (L, 8, 192, 68, wo.WRAP_X) if axis == "x" else (128, L, 128, 192, wo.WRAP_Y)
    c = case(*geom, ov=64, bs=64, N=1, C=2)
    n = c.g.cols if axis == "x" else c.g.rows
    assert n == 256 and c.g.overlap == 64 and max(c.g.xs[c.g.cols - 1], c.g.ys[c.g.rows - 1]) == 32632
    run_all(c, "f16", expect=vector("f16"))
    run_blend(c, "md", "f16", flags=FORCE_GENERIC)
    past = (16448, 8, 128, 68) if axis == "x" else (8, 16448, 68, 128)   # stride 64: ceil(16448 / 64) = 257
    with pytest.raises(TdError) as e:
        engine.make_grid(*past, 64, 4, wrap=wo.WRAP_X if axis == "x" else wo.WRAP_Y)
    assert e.value.status == TD_ERR_UNSUPPORTED and "TD_MAX_GRID_DIM" in str(e.value)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", ["x", "y"])
def test_canvas_extent_32767_runs_and_32768_is_refused(axis):
    """Origins travel to the kernels as `short`: a 32767-long periodic axis runs (x: generic, an odd width; y: vector),
    a 32768-long one is refused by the entries' plan check before anything launches."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_UNSUPPORTED, TdError
    geom = (32767, 8, 192, 68, wo.WRAP_X) if axis == "x" else (128, 32767, 128, 192, wo.WRAP_Y)
    c = case(*geom, ov=64, bs=64, N=1, C=2)
    assert max(c.g.cols, c.g.rows) == 256
    for dn in ("f16", "f32"):
        run_all(c, dn, expect=generic(dn) if axis == "x" else vector(dn))
    big = Case(*((32768, 8, 192, 68, wo.WRAP_X) if axis == "x" else (128, 32768, 128, 192, wo.WRAP_Y)), ov=64, bs=256, N=1, C=1)
    x = torch.zeros(big.shape, dtype=torch.float16, device="cuda")
    tiles = torch.zeros((big.T, 1, big.th, big.tw), dtype=torch.float16, device="cuda")
    w = torch.ones((big.H, big.W), device="cuda")
    for call in (lambda: engine.scatter_tiles(big.g, x),
                 lambda: engine.blend_multidiffusion(big.g, [tiles], 1, 1, big.T, w, torch.float16),
                 lambda: engine.blend_mixture(big.g, [tiles], 1, 1, big.T, torch.ones((big.th, big.tw), device="cuda"), w, x)):
        with pytest.raises(TdError) as e:
            call()
        assert e.value.status == TD_ERR_UNSUPPORTED and "too large" in str(e.value)


@pytest.mark.gpu
def test_65535_planes_run_on_the_vector_forms_and_65536_are_refused():
    """N*C = 65535 is the vector blend's grid.z; an 8 x 8 canvas wrapped in y (two tile rows, one crossing the seam)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_UNSUPPORTED, TdError
    c = case(8, 8, 8, 6, wo.WRAP_Y, ov=2, bs=2, N=5, C=13107)
    assert c.N * c.C == 65535 and list(c.g.ys[:c.g.rows]) == [0, 4]
    run_all(c, "f16", expect=vector("f16"))
    N, C = 4, 16384
    x = torch.zeros((N, C, 8, 8), dtype=torch.float16, device="cuda")
    tiles = torch.zeros((c.T * N, C, c.th, c.tw), dtype=torch.float16, device="cuda")
    w = torch.from_numpy(c.weights).cuda()
    for call in (lambda: engine.scatter_tiles(c.g, x),
                 lambda: engine.blend_multidiffusion(c.g, [tiles], N, C, c.T, w, torch.float16),
                 lambda: engine.blend_mixture(c.g, [tiles], N, C, c.T, torch.from_numpy(c.tile_weights).cuda(), w, x)):
        with pytest.raises(TdError) as e:
            call()
        assert e.value.status == TD_ERR_UNSUPPORTED and "N*C" in str(e.value)


@pytest.mark.gpu
def test_128_batch_tensors_and_129():
    """128 tile-batch tensors go to the kernel in one pointer table; 129 are refused by the C-ABI and merged by the engine."""
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    c = case(128, 64, 16, 16, WRAP_XY, ov=8, bs=1)
    assert len(c.batched) == c.g.num_batches == _cabi.TD_MAX_BATCH_PTRS
    for op in ("md", "mod"):
        assert run_blend(c, op, "f16") == {vec_form(op, "f16")}
    big = case(136, 64, 16, 16, WRAP_XY, ov=8, bs=1)
    assert len(big.batched) == 136
    douts = [o.cuda() for o in big.outs("f16")]
    ptrs = (ctypes.c_void_p * 129)(*[o.data_ptr() for o in douts[:129]])
    out = torch.empty(big.shape, device="cuda")
    st = _cabi.lib.td_blend_multidiffusion(ctypes.byref(big.g), ptrs, 129, 1, big.N, big.C, _cabi.TD_F16, _cabi.TD_F16,
                                           torch.from_numpy(big.weights).cuda().data_ptr(), None, out.data_ptr(), None, 0, None)
    assert st == _cabi.TD_ERR_UNSUPPORTED and b"TD_MAX_BATCH_PTRS" in _cabi.lib.td_last_error()
    for op in ("md", "mod"):
        assert run_blend(big, op, "f16") == {vec_form(op, "f16")}


@pytest.mark.gpu
@pytest.mark.parametrize("dn", ["f16", "bf16"])
def test_36_visits_per_pixel(dn):
    """Periodic tile 24, overlap 20 on both axes: every pixel is covered by 6 x 6 tiles, added in tile order with one
    rounding per add in the 16-bit canvas dtype."""
    c = case(48, 48, 24, 24, WRAP_XY, ov=20, bs=16, N=1, C=4)
    assert c.weights.min() == c.weights.max() == 36
    run_all(c, dn, expect=vector(dn))
    run_all(c, dn, FORCE_GENERIC, expect=generic(dn))


# tiles as wide and as tall as the canvas, three origins each: every canvas vector holding an origin also holds the
# last columns of that tile, reached after the seam
FULL = (64, 24, 64, 24, WRAP_XY, (0, 21, 45), (0, 7, 13))
# origins far from the search estimate (floor(k L / n) for a periodic axis): clustered, equal neighbours, a bounded y
CLUSTERED = {"clustered": (64, 24, 56, 20, WRAP_XY, (0, 1, 2, 3, 59), (0, 1, 2, 21)),
             "equal_neighbours": (64, 24, 56, 20, WRAP_XY, (0, 0, 3, 3, 59), (0, 0, 20, 20)),
             "bounded_y": (64, 24, 56, 20, wo.WRAP_X, (0, 1, 2, 3, 59), (0, 1, 2, 4))}
HAND = {"canvas_wide_and_tall": FULL, **CLUSTERED}


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("plan", list(HAND))
def test_hand_made_periodic_plans(plan, dn):
    W, H, tw, th, wrap, xs, ys = HAND[plan]
    c = case(W, H, tw, th, wrap, bs=5, xs=xs, ys=ys)
    assert c.weights.min() >= 1
    run_all(c, dn, expect=vector(dn))
    run_all(c, dn, FORCE_GENERIC, expect=generic(dn))


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_tiny_canvases(dn):
    """W = one vector, H = 1: periodic 1 x 1 tiles (generic), and one-vector tiles at three origins (vector, every
    canvas vector straddling two of them)."""
    vec = 16 // DTYPES[dn].itemsize
    c = case(vec, 1, 1, 1, WRAP_XY, ov=0, bs=3)
    assert (c.g.cols, c.g.rows, c.tw, c.th) == (vec, 1, 1, 1)
    run_all(c, dn, expect=generic(dn))
    c = case(vec, 1, vec, 1, WRAP_XY, bs=2, xs=(0, 1, vec - 1), ys=(0,))
    run_all(c, dn, expect=vector(dn))


@pytest.mark.gpu
@pytest.mark.parametrize("dn", ["f16", "f32"])
def test_scatter_sub_ranges(dn):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    c = case(*BASE, ov=8)
    for rng in ((0, 1), (c.T - 1, c.T), (5, 9)):
        for flags in (0, FORCE_GENERIC):
            got = run_scatter(c, dn, flags, rng=rng)
            assert got == {(vec_form if flags == 0 else generic_form)("scatter", dn)}, (rng, flags, got)
    empty = engine.scatter_tiles(c.g, c.x(dn).cuda(), tile_begin=7, tile_end=7)
    torch.cuda.synchronize()
    assert tuple(empty.shape) == (0, c.C, c.th, c.tw)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the bit checks catch injected kernel defects (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _accumulate(outs, batched, N, shape, dtype, defect=None, mod=None, vec=8):
    """The wrap oracle's accumulator written out column by column, with an optional defect of a kernel:
    no_range_b      -- tiles that reach a pixel only after the seam are skipped
    no_second_visit -- a tile as wide as the canvas loses the columns before its origin in the vector holding it
    fp32_acc        -- 16-bit values accumulated in fp32 and rounded once at the end
    product_order   -- MoD computes (tile * tile_weights) * rescale
    `mod`: (tile_weights, rescale) for Mixture of Diffusers."""
    H, W = shape[2], shape[3]
    acc = torch.zeros(shape, dtype=torch.float32 if defect == "fp32_acc" else dtype)
    for out, bbs in zip(outs, batched):
        for i, (x, y, w, h) in enumerate(bbs):
            t = out[i * N:(i + 1) * N]
            u = torch.arange(w)
            keep = torch.ones(w, dtype=torch.bool)
            if defect == "no_range_b":
                keep &= x + u < W
            if defect == "no_second_visit" and w == W and x % vec:
                keep &= ~(((x + u) % W >= x - x % vec) & ((x + u) % W < x))
            cols = ((x + u) % W)[keep]
            rows = (y + torch.arange(h)) % H
            idx = (slice(None), slice(None), rows[:, None], cols[None, :])
            tk = t[:, :, :, keep]
            if mod is None:
                acc[idx] = acc[idx] + tk
            else:
                tw = torch.from_numpy(mod[0])[:, keep]
                rs = torch.from_numpy(mod[1])[rows[:, None], cols[None, :]]
                val = (tk * tw) * rs if defect == "product_order" else tk * (tw * rs)
                acc[idx] = (acc[idx] + val).to(acc.dtype)
    return acc.to(dtype)


DEFECTS = {  # defect -> (plan, dtype, mode): the geometry each defect is aimed at
    "no_range_b": ((120, 64, 40, 24, wo.WRAP_X, 8, None, None), "f32", "md"),
    "no_second_visit": ((64, 24, 64, 24, WRAP_XY, None, (0, 21, 45), (0, 7, 13)), "f16", "md"),
    "fp32_acc": ((48, 48, 24, 24, WRAP_XY, 20, None, None), "f16", "md"),
    "product_order": ((120, 64, 40, 24, WRAP_XY, 8, None, None), "f32", "mod"),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_checks_catch_injected_defects(defect):
    """The column-by-column accumulator equals the oracle's bits without a defect and differs with the one aimed at this
    geometry: a kernel with that defect fails the bit checks above."""
    (W, H, tw, th, wrap, ov, xs, ys), dn, mode = DEFECTS[defect]
    c = Case(W, H, tw, th, wrap, ov=ov, bs=5, xs=xs, ys=ys, N=1, C=2)
    dt = DTYPES[dn]
    outs = c.outs(dn)
    mod = (c.tile_weights, c.rescale) if mode == "mod" else None
    want = c.want(mode, dn, dn)
    want = want[1] if mode == "md" else want
    assert_bit_equal(_accumulate(outs, c.batched, c.N, c.shape, dt, mod=mod), want, "faithful restatement")
    bad = _accumulate(outs, c.batched, c.N, c.shape, dt, defect=defect, mod=mod)
    assert not np.array_equal(bad.view(torch.int16 if dt.itemsize == 2 else torch.int32).numpy(),
                              want.view(torch.int16 if dt.itemsize == 2 else torch.int32).numpy()), f"{defect} goes unnoticed"


# ---------------------------------------------------------------------------------------------------------------------
# 5. origins out of order are refused by every grid entry (CPU: null tensors, nothing can launch)
# ---------------------------------------------------------------------------------------------------------------------
ENTRIES = ["td_scatter_tiles", "td_blend_multidiffusion", "td_blend_mixture", "td_blend_multidiffusion_rows", "td_blend_mixture_rows",
           "td_blend_multidiffusion_wrap_rows", "td_blend_mixture_wrap_rows", "td_blend_multidiffusion_peer"]


def _call_with_nulls(lib, entry, g):
    """`entry` on plan `g` with every tensor, the batch table and the wait table null."""
    F16 = 0
    gp = ctypes.byref(g)
    if entry == "td_scatter_tiles":
        return lib.td_scatter_tiles(gp, None, None, 2, 4, F16, 0, g.num_tiles, 0, None)
    head = (gp, None, g.num_batches, g.tile_bs, 2, 4, F16, F16)
    if entry == "td_blend_multidiffusion":
        return lib.td_blend_multidiffusion(*head, None, None, None, None, 0, None)
    if entry == "td_blend_mixture":
        return lib.td_blend_mixture(*head, None, None, None, 0, None)
    if entry == "td_blend_multidiffusion_rows":
        return lib.td_blend_multidiffusion_rows(*head, None, None, None, None, 0, 8, None, 0, None, 0, 0, 0, None)
    if entry == "td_blend_mixture_rows":
        return lib.td_blend_mixture_rows(*head, None, None, None, 0, 8, None, 0, None, 0, 0, 0, None)
    if entry == "td_blend_multidiffusion_wrap_rows":
        return lib.td_blend_multidiffusion_wrap_rows(*head, None, None, None, 0, 8, None, 0, None, 0, 0, 0, None)
    if entry == "td_blend_mixture_wrap_rows":
        return lib.td_blend_mixture_wrap_rows(*head, None, None, None, 0, 8, None, 0, None, 0, 0, 0, None)
    return lib.td_blend_multidiffusion_peer(*head, None, None, None, None, 1, None, 0, None)


@pytest.mark.parametrize("wrap", [0, WRAP_XY], ids=["bounded", "wrapped"])
@pytest.mark.parametrize("axis", ["xs", "ys"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_out_of_order_origins_are_refused(entry, axis, wrap):
    """Every origin search assumes non-decreasing origins.  Two swapped neighbours (both still inside the canvas) are
    refused with TD_ERR_INVALID_ARG and a message naming the axis and the index; equal neighbours pass the check (the call
    then fails on its null pointers, as it does with a plan in order)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, lib
    g = engine.make_grid(64, 48, 16, 16, 8, 4, wrap=wrap)
    origins = getattr(g, axis)
    assert (g.cols if axis == "xs" else g.rows) > 3
    origins[1], origins[2] = origins[2], origins[1]
    assert _call_with_nulls(lib, entry, g) == TD_ERR_INVALID_ARG
    msg = lib.td_last_error().decode()
    assert "out of order" in msg and f"{axis}[2]=" in msg, msg
    origins[2] = origins[1]
    assert _call_with_nulls(lib, entry, g) == TD_ERR_INVALID_ARG
    assert "out of order" not in lib.td_last_error().decode()


@pytest.mark.parametrize("wrap", [0, WRAP_XY], ids=["bounded", "wrapped"])
def test_empty_scatter_range_launches_nothing(wrap):
    """A tile shard without tiles scatters [b, b): its output tensor is empty (null data pointer), and nothing launches.
    The range and the dtype are still checked."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, TD_F16, TD_OK, lib
    g = engine.make_grid(64, 48, 16, 16, 8, 4, wrap=wrap)
    for b in (0, 5, g.num_tiles):
        assert lib.td_scatter_tiles(ctypes.byref(g), None, None, 2, 4, TD_F16, b, b, 0, None) == TD_OK
    assert lib.td_scatter_tiles(ctypes.byref(g), None, None, 2, 4, TD_F16, g.num_tiles + 1, g.num_tiles + 1, 0, None) == TD_ERR_INVALID_ARG
    assert lib.td_scatter_tiles(ctypes.byref(g), None, None, 2, 4, 7, 5, 5, 0, None) == TD_ERR_INVALID_ARG
    assert lib.td_scatter_tiles(ctypes.byref(g), None, None, 2, 4, TD_F16, 0, 1, 0, None) == TD_ERR_INVALID_ARG
