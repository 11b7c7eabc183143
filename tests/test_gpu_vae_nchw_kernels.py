"""The NCHW tiled-VAE kernels (csrc/td_vae.cu: td_gn_stats, td_gn_apply, td_copy_region, td_resample_nearest,
td_affine_clamp) against float64 and eager torch, at every template instantiation the host can launch, at the host-side
grid and chunk limits, and end to end through fast mode.  These kernels do GroupNorm for every fp32 autoencoder (the
module backend), the tile crop / paste / wrap-around load of that backend, and the fast-mode estimator input of both
backends (and DemoFusion's re-standardisation).

Which form ran is asserted from a CUPTI kernel trace (`launched` / `template_args`), in a fresh interpreter (see
`_forms`).  References are computed in float64
on the device from the exact inputs.  Bounds (u = 2^-24, the fp32 unit roundoff; U / TAU: unit roundoff and half the
smallest subnormal spacing of the output format: fp16 2^-11 / 2^-25, bf16 2^-8 / 2^-134, fp32 2^-24 / 2^-150):

  gn_stats   Plan (`plan_stats`, a port of the host code): a segment of n elements is cut into `chunks` chunks of `chunk`
             elements (a multiple of the vector width v = 16 / element size), one 256-thread CTA per chunk.  Every thread
             sums d = x - k over at most n_t = ceil(chunk / (256 v)) v elements (n_t = ceil(chunk / 256) on the scalar
             path), k being the chunk's first element; the per-thread moments (count, mean, M2) are then merged with
             Chan's update through a 5-level warp tree, a 3-level tree over the CTA's 8 warps, ceil(chunks / 32) serial
             merges per lane of the final warp and its 5-level tree: depth D = 13 + ceil(chunks / 32).
             With mu, M2 the float64 mean and sum of squared deviations, R = max |x - mu| (every partial mean lies in
             [mu - R, mu + R], every |d| <= 2R) and S = sum (x - k)^2:
               e_mean = u [(D + 2)(|mu| + R) + (n_t + 3 D) 2R]
                 (one rounding of x - k and of the running sum per element, of k + s / n per thread, and of
                 a.mean + d f per merge)
               e_M2   = u (n_t + 4 + 4 D)(S + M2) + 4 D n R e_mean
                 (the fma'd sum of squares and ss - s * md per thread; 4 roundings per merge; and the d^2 n_a n_b / n
                 merge terms with d off by at most 2 e_mean: each element takes part in D merges, so
                 sum n_a n_b / n <= n D / 2)
               var = M2 / n (biased) or M2 / (n - 1) (unbiased): e_var = e_M2 / n' + u var.
             ASSUMPTIONS: first order in u (the O(u^2) terms are dropped); counts travel as float and are exact because
             every partial count is a multiple of v below 2^24 per thread, and their sums stay multiples of v (checked
             past 2^24 elements by the 1024-chunk cases).  The bound is loose where |mu| >> R (the merge terms carry
             mean roundings of u |mu|); structural defects are caught by the probes instead.  min / max are bit-exact.
             An unbiased segment of one element returns var 0 (torch: NaN); fast mode never issues one (the estimator's
             long side is the tile size), so it is not tested.
  gn_apply   t = fmaf(x, A, fmaf(-mu, A, beta)), A = gamma / sqrt(var + eps) (5 roundings: 10 u relative after the fma
             with gamma): e_t = 10 u (|x A| + |mu A|) + u (|mu A| + |beta|) + u |t| -- outputs near zero are pure
             cancellation of x A against mu A - beta, so the bound carries those magnitudes, not |t|.  SiLU as in
             test_gpu_vae_kernels.py (`_silu_err`, __expf / __fdividef, 0 below t = -87.3).  Output: U |ref| + (1 + U) e + TAU.
  copy, resample  bit-exact (16-bit types move as opaque words: NaN payloads, -0.0 and subnormals survive).
  affine_clamp    bit-exact against the eager CUDA sequence ((x - mn) / sn * so + mo).clamp_(lo, hi) in the tensor dtype.
"""
import copy
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from helpers import assert_bit_equal
from test_gpu_blend_limits import launched, template_args
from test_gpu_vae_kernels import _silu_err

DTS = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
DN = list(DTS)
CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}
ES = {torch.float16: 2, torch.bfloat16: 2, torch.float32: 4}
TNAME = {torch.float16: "__half", torch.bfloat16: "__nv_bfloat16", torch.float32: "float"}
WORD = {torch.float16: "__half", torch.bfloat16: "__half", torch.float32: "float"}     # copy / resample move words
INT = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
TAU = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 2.0 ** -150}
E32 = 2.0 ** -24
WORST = {}          # (family, dtype name) -> worst err / bound seen

K_STATS, K_APPLY, K_COPY, K_RESAMPLE, K_CLAMP = ("gn_stats_partial_kernel", "gn_apply_kernel", "copy_region_kernel",
                                                 "resample_kernel", "affine_clamp_kernel")
OK, INVALID, UNSUPPORTED, CAPACITY = 0, -1, -2, -4


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def _tv():
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    return tilevae


def _stream():
    return _cabi().current_stream_ptr() if torch.cuda.is_available() else None


def _dn(dt):
    return next(k for k, v in DTS.items() if v == dt)


def _note(family, dt, ratio):
    key = (family, _dn(dt))
    WORST[key] = max(WORST.get(key, 0.0), ratio)


def _randn(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * scale + shift


def _bits(n, dt, seed):
    """n random bit patterns of dtype dt (every class: NaN payloads, +-inf, +-0, subnormals)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = INT[dt]
    info = torch.iinfo(w)
    return torch.randint(info.min, info.max, (n,), generator=g, device="cuda", dtype=torch.int64).to(w).view(dt)


# Which kernel ran is read from a CUPTI trace, and that trace is reliable only in a young process: late in a long GPU
# session (hundreds of earlier profiler sessions, several minutes in) most sessions come back without kernel records
# whatever the device memory or the session length.  So the form assertions run in a fresh interpreter
# (`test_launched_forms_in_a_fresh_process` runs the tests that make them there), and in this process `_forms` only
# runs the call; every numerical check runs in both.
FORMS_CHILD = os.environ.get("TD_NCHW_FORMS_CHILD") == "1"


class _NotTraced:
    """What `_forms` returns outside the child interpreter: equal to any expected form set (the child asserts it)."""

    def __eq__(self, other):
        return True

    __hash__ = None

    def __repr__(self):
        return "<forms asserted in the child interpreter>"


def _forms(fn, kernel):
    """Template arguments of every `kernel` instantiation `fn` launched (in the child interpreter; see above)."""
    if not FORMS_CHILD:
        fn()
        return _NotTraced()
    return {tuple(a) for a in template_args(launched(fn), kernel)}


FORM_TESTS = ("every_form or grid_and_plane_limits or copy_region_vector or copy_region_grid or resample_nearest_bit "
              "or affine_clamp_matches")


@pytest.mark.gpu
def test_launched_forms_in_a_fresh_process():
    """The tests that assert which template ran, rerun in a fresh interpreter where the kernel trace is complete."""
    if FORMS_CHILD:
        pytest.skip("already the child interpreter")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    cmd = [sys.executable, *flags, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k", FORM_TESTS]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(cmd, cwd=root, env=dict(os.environ, TD_NCHW_FORMS_CHILD="1"), capture_output=True, text=True, timeout=1200)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail


# ---------------------------------------------------------------------------------------------------------------------
# port of the host plan of td_gn_stats (csrc/td_vae.cu, plan_stats)
# ---------------------------------------------------------------------------------------------------------------------
STAT_THREADS, SMS = 256, 148


def plan_stats(nseg, seg_len, es, aligned=True):
    """-> (chunk, chunks, vector path).  ~64 KB per CTA, at least ~4 CTAs per SM overall, at most 1024 chunks per
    segment; the chunk is rounded up to the vector width whether or not the vector path runs."""
    vec = 16 // es
    chunk = 65536 // es
    chunks = -(-seg_len // chunk)
    want = -(-(SMS * 4) // nseg)
    if chunks < want:
        chunks = min(want, max(1, seg_len // (STAT_THREADS * vec)))
    chunks = max(1, min(chunks, 1024))
    chunk = -(-seg_len // chunks)
    chunk = -(-chunk // vec) * vec
    return chunk, -(-seg_len // chunk), aligned and seg_len % vec == 0


def workspace_bytes(nseg, seg_len, es):
    return nseg * plan_stats(nseg, seg_len, es)[1] * 5 * 4


# (nseg, seg_len, element size) -> (chunk, chunks): every branch of the plan, computed by hand
PLAN_CASES = [
    ((1, 1000, 4), (1000, 1)),               # one chunk: seg_len < 256 v
    ((1, 5000, 4), (1252, 4)),               # too few segments: seg_len / (256 v) = 4 chunks, last one partial (1244)
    ((2, 1_000_000, 4), (3380, 296)),        # want-limited: ceil(592 / 2) = 296 chunks, last one 2900
    ((64, 200_000, 4), (15388, 13)),         # chunk-size-limited: ceil(200000 / 16384) = 13 >= want 10, last 15344
    ((1, 1024 * 16384 + 4, 4), (16388, 1024)),      # 1024 cap, fp32 (> 2^24 elements), last chunk 12296
    ((1, 1024 * 32768 + 8, 2), (32776, 1024)),      # 1024 cap, 16-bit (> 2^25 elements), last chunk 24592
    ((1, 1024 * 32768 + 3, 2), (32776, 1024)),      # same plan on the scalar path (seg_len % 8 != 0)
    ((65535, 8, 2), (8, 1)),                 # the grid limit of segments: one chunk each
]


@pytest.mark.parametrize("args,want", PLAN_CASES, ids=[f"{a[0]}x{a[1]}x{a[2]}" for a, _ in PLAN_CASES])
def test_plan_stats_port_matches_hand_computed_plans(args, want):
    nseg, seg_len, es = args
    chunk, chunks, _ = plan_stats(nseg, seg_len, es)
    assert (chunk, chunks) == want
    vec = 16 // es
    assert chunk % vec == 0 and (chunks - 1) * chunk < seg_len <= chunks * chunk
    assert chunks <= 1024
    # the partial counts the kernel carries as float are exact: per-thread counts are below 2^24 and every sum of
    # chunk counts is a multiple of the vector width that fits in 24 + log2(v) bits
    per_thread = -(-chunk // (STAT_THREADS * vec)) * vec
    assert per_thread < 2 ** 24
    if seg_len % vec == 0:
        # vector path: every partial count (whole chunks, the last one partial) is a multiple of v below 2^24 v, so
        # fp32 holds it exactly even past 2^24 elements
        totals = [k * chunk for k in range(1, chunks)] + [seg_len]
        assert all(t % vec == 0 and t < 2 ** 24 * vec for t in totals)
        assert all(float(torch.tensor(t, dtype=torch.float32).item()) == t for t in totals)


# ---------------------------------------------------------------------------------------------------------------------
# float64 references and bounds
# ---------------------------------------------------------------------------------------------------------------------
def _stats64(x, nseg, seg_len, unbiased, aligned=True):
    """float64 (mean, var, min, max) of every segment and the bounds of the module docstring."""
    es = x.element_size()
    chunk, chunks, vec_path = plan_stats(nseg, seg_len, es, aligned)
    vec = 16 // es
    n_t = -(-chunk // (STAT_THREADS * vec)) * vec if vec_path else -(-chunk // STAT_THREADS)
    D = 13 + -(-chunks // 32)
    xs = x.reshape(nseg, seg_len).double()
    mu = xs.mean(1)
    dev = xs - mu[:, None]
    m2 = (dev * dev).sum(1)
    R = dev.abs().amax(1)
    del dev
    k = xs[:, ::chunk].repeat_interleave(chunk, dim=1)[:, :seg_len]
    sh = xs - k
    del k
    S = (sh * sh).sum(1)
    del sh
    var, e_mean, e_var = _stats_bounds(mu, m2, R, S, seg_len, n_t, D, unbiased)
    return mu, var, xs.amin(1), xs.amax(1), e_mean, e_var


def _stats_bounds(mu, m2, R, S, n, n_t, D, unbiased, merge_roundings=(3, 4)):
    """(var, e_mean, e_var) of the module docstring from the float64 moments of each segment (n elements, at most n_t
    per thread, merge depth D).  merge_roundings: the roundings per merge in the mean and M2 terms (3 and 4 here)."""
    rm, rq = merge_roundings
    u = E32
    e_mean = u * ((D + 2) * (mu.abs() + R) + (n_t + rm * D) * 2 * R)
    e_m2 = u * (n_t + 4 + rq * D) * (S + m2) + 4 * D * n * R * e_mean
    nd = n - 1 if unbiased else n
    var = m2 / max(nd, 1)
    e_var = e_m2 / max(nd, 1) + u * var
    return var, e_mean, e_var


def _check_stats(x, nseg, seg_len, unbiased, what, minmax=True, aligned=True):
    """td_gn_stats through tilevae._segment_stats against float64; returns the launched (T, VECTOR, MINMAX) forms."""
    tv = _tv()
    box = {}

    def run():
        box["r"] = tv._segment_stats(x, nseg, seg_len, unbiased=unbiased, want_minmax=minmax)
    forms = _forms(run, K_STATS)
    out = box["r"]
    var, mean = out[0], out[1]
    mu, v64, lo, hi, e_mean, e_var = _stats64(x, nseg, seg_len, unbiased, aligned)
    dt = x.dtype
    assert torch.isfinite(mean).all() and torch.isfinite(var).all(), f"{what}: non-finite statistics"
    assert (var >= 0).all(), f"{what}: negative variance"
    rm = ((mean.double() - mu).abs() / e_mean.clamp_min(1e-300)).max().item()
    rv = ((var.double() - v64).abs() / e_var.clamp_min(1e-300)).max().item()
    _note("gn_stats", dt, max(rm, rv))
    assert rm <= 1 and rv <= 1, f"{what}: mean err/bound {rm:.3g}, var err/bound {rv:.3g}"
    if minmax:
        assert torch.equal(out[2].double(), lo) and torch.equal(out[3].double(), hi), f"{what}: min / max not exact"
    return forms


def _apply64(x, mean, var, gamma, beta, act, groups, per_batch, eps=1e-6):
    """float64 reference and bound of td_gn_apply for x [B, C, L] (see the module docstring)."""
    dt = x.dtype
    B, C = x.shape[:2]
    cpg = C // groups
    m = mean.double().view(B if per_batch else 1, groups).repeat_interleave(cpg, 1)
    v = var.double().view(B if per_batch else 1, groups).repeat_interleave(cpg, 1)
    A = 1.0 / torch.sqrt(v + float(torch.tensor(eps, dtype=torch.float32)))
    if gamma is not None:
        A = A * gamma.double()
    be = beta.double().expand(m.shape) if beta is not None else torch.zeros_like(m)
    A, m, be = A[..., None], m[..., None], be[..., None]
    xd = x.double()
    xa, ma = xd * A, m * A
    t = xa - ma + be
    u = E32
    e_t = 10 * u * (xa.abs() + ma.abs()) + u * (ma.abs() + be.abs()) + u * t.abs()
    if act:
        z = t * torch.sigmoid(t)
        e = 1.1 * e_t + _silu_err(t, z)
    else:
        z, e = t, e_t
    return z, U[dt] * z.abs() + (1.0 + U[dt]) * e + TAU[dt]


def _within(got, ref, bound, family, dt, what):
    g = got.double()
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    ratio = (g - ref).abs() / bound
    worst = ratio.max().item()
    _note(family, dt, worst)
    if worst > 1.0:
        i = int(ratio.argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        n = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n} elements over the bound; worst at {idx}: got {g[idx].item()!r} ref {ref[idx].item()!r} "
                             f"bound {bound[idx].item():.3g} (err / bound {worst:.3g})")
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the checkers catch the defects they are meant to catch
# ---------------------------------------------------------------------------------------------------------------------
def _stats_ok(vals, x, nseg, seg_len, unbiased):
    mu, v64, _, _, e_mean, e_var = _stats64(x, nseg, seg_len, unbiased)
    mean, var = vals
    return bool(((mean - mu).abs() <= e_mean).all() and ((var - v64).abs() <= e_var).all())


def _probe_ok(mean, var, c, delta, n, unbiased):
    want_v = delta * delta / n if unbiased else delta * delta * (n - 1) / n / n
    return abs((mean - c) / (delta / n) - 1) <= 1e-3 and abs(var / want_v - 1) <= 1e-3


def test_checkers_reject_injected_defects():
    """Each checker, fed float64 results of a deliberately wrong algorithm, must fail: a dropped element, a duplicated
    vector and a wrong shift against the statistics bound and the probe rule; a wrong batch index against the apply
    bound.  The correct float64 result passes each check."""
    g = torch.Generator().manual_seed(7)
    nseg, n = 3, 4096
    x = (torch.randn(nseg * n, generator=g) * 1.3 + 0.4).float()
    xs = x.double().view(nseg, n)
    chunk = plan_stats(nseg, n, 4)[0]
    assert chunk < n

    def moments(rows):
        return torch.stack([r.mean() for r in rows]), torch.stack([r.var() for r in rows])
    assert _stats_ok(moments(list(xs)), x, nseg, n, True)
    far = int((xs[0] - xs[0].mean()).abs().argmax())
    dropped = [torch.cat([xs[0][:far], xs[0][far + 1:]]), xs[1], xs[2]]
    v0 = far // 4 * 4
    duplicated = [torch.cat([xs[0], xs[0][v0:v0 + 4]]), xs[1], xs[2]]
    # a wrong shift: chunk 1 adds back chunk 0's shift k instead of its own
    wrong = xs[0].clone()
    wrong[chunk:2 * chunk] += xs[0][0] - xs[0][chunk]
    assert not _stats_ok(moments(dropped), x, nseg, n, True)
    assert not _stats_ok(moments(duplicated), x, nseg, n, True)
    assert not _stats_ok(moments([wrong, xs[1], xs[2]]), x, nseg, n, True)
    # probes: constant c with one element c + delta; a dropped or duplicated vector holding it is off by 100 %
    c, delta, m = 2.0 ** -10, 2.0 ** -3, 32768
    seg = torch.full((m,), c, dtype=torch.float64)
    seg[m - 1] = c + delta
    assert _probe_ok(seg.mean().item(), seg.var().item(), c, delta, m, True)
    lost = seg[:-8]
    assert not _probe_ok(lost.mean().item(), lost.var().item(), c, delta, m, True)
    dup = torch.cat([seg, seg[-8:]])
    assert not _probe_ok(dup.mean().item(), dup.var().item(), c, delta, m, True)
    bled = seg.clone()
    bled[0] = c + delta      # the next segment's probe read into this one
    assert not _probe_ok(bled.mean().item(), bled.var().item(), c, delta, m, True)
    # apply: statistics of batch b taken from batch b - 1
    B, C, L, groups = 3, 8, 64, 4
    xa = torch.randn((B, C, L), generator=g).float()
    mean = torch.randn(B * groups, generator=g).float()
    var = torch.rand(B * groups, generator=g).float() + 0.5
    ref, bound = _apply64(xa, mean, var, None, None, False, groups, True)
    assert ((ref - ref).abs() <= bound).all()
    wrong, _ = _apply64(xa, mean.view(B, groups).roll(1, 0).reshape(-1), var.view(B, groups).roll(1, 0).reshape(-1), None, None,
                        False, groups, True)
    assert ((wrong - ref).abs() > bound).any()


# ---------------------------------------------------------------------------------------------------------------------
# refusals: every argument check of the five entry points (no launch, so no device needed)
# ---------------------------------------------------------------------------------------------------------------------
P = 1 << 20          # a 16-byte-aligned address that is never dereferenced: every case below returns before a launch


def _err():
    return _cabi().lib.td_last_error().decode()


def test_gn_stats_refusals():
    lib = _cabi().lib
    ws = workspace_bytes(4, 1000, 4)
    good = dict(x=P, nseg=4, seg_len=1000, dtype=2, unbiased=0, ws=P, wsb=ws, mean=P, var=P, lo=None, hi=None)
    cases = [("x", dict(x=None), INVALID), ("mean", dict(mean=None), INVALID), ("var", dict(var=None), INVALID),
             ("workspace", dict(ws=None), INVALID), ("nseg 0", dict(nseg=0), INVALID), ("nseg -1", dict(nseg=-1), INVALID),
             ("seg_len 0", dict(seg_len=0), INVALID), ("seg_len -5", dict(seg_len=-5), INVALID), ("dtype 3", dict(dtype=3), INVALID),
             ("dtype -1", dict(dtype=-1), INVALID), ("65536 segments", dict(nseg=65536, wsb=1 << 40), UNSUPPORTED),
             ("workspace one byte short", dict(wsb=ws - 1), CAPACITY),
             ("planned workspace of 65535 segments one byte short", dict(nseg=65535, seg_len=8, dtype=0, wsb=workspace_bytes(65535, 8, 2) - 1),
              CAPACITY)]
    for name, over, want in cases:
        a = {**good, **over}
        st = lib.td_gn_stats(a["x"], a["nseg"], a["seg_len"], a["dtype"], a["unbiased"], a["ws"], a["wsb"], a["mean"], a["var"], a["lo"],
                             a["hi"], None)
        assert st == want, f"{name}: status {st} ({_err()})"
    assert lib.td_gn_stats_workspace_bytes(65535, 8, 0) == 65535 * 1024 * 20      # the upper bound the wrapper allocates
    for args in [(0, 8, 0), (4, 0, 0), (4, 8, 7)]:
        assert lib.td_gn_stats_workspace_bytes(*args) == 0


def test_gn_apply_refusals():
    lib = _cabi().lib
    good = dict(x=P, y=P, B=2, C=64, HW=100, dtype=2, groups=32, mean=P, var=P)
    cases = [("x", dict(x=None), INVALID), ("y", dict(y=None), INVALID), ("mean", dict(mean=None), INVALID),
             ("var", dict(var=None), INVALID), ("B 0", dict(B=0), INVALID), ("C 0", dict(C=0), INVALID), ("HW 0", dict(HW=0), INVALID),
             ("HW -1", dict(HW=-1), INVALID), ("groups 0", dict(groups=0), INVALID), ("C % groups", dict(C=48), INVALID),
             ("dtype 3", dict(dtype=3), INVALID), ("B*C = 65536", dict(B=2, C=32768), UNSUPPORTED),
             ("B*C = 65536 (one batch)", dict(B=1, C=65536, groups=64), UNSUPPORTED)]
    for name, over, want in cases:
        a = {**good, **over}
        st = lib.td_gn_apply(a["x"], a["y"], a["B"], a["C"], a["HW"], a["dtype"], a["groups"], a["mean"], a["var"], 0, None, None,
                             1e-6, 0, None)
        assert st == want, f"{name}: status {st} ({_err()})"


def test_copy_region_refusals():
    lib = _cabi().lib
    good = dict(src=P, dst=P, planes=2, rows=3, cols=8, dtype=0)
    cases = [("src", dict(src=None), INVALID), ("dst", dict(dst=None), INVALID), ("planes -1", dict(planes=-1), INVALID),
             ("rows -1", dict(rows=-1), INVALID), ("cols -1", dict(cols=-1), INVALID), ("dtype 3", dict(dtype=3), INVALID),
             ("65536 planes", dict(planes=65536), UNSUPPORTED),
             ("zero planes", dict(planes=0), OK), ("zero rows", dict(rows=0), OK), ("zero cols", dict(cols=0), OK),
             ("zero size and 65536 planes", dict(planes=65536, rows=0), OK)]
    for name, over, want in cases:
        a = {**good, **over}
        st = lib.td_copy_region(a["src"], a["dst"], a["planes"], a["rows"], a["cols"], 24, 8, 24, 8, a["dtype"], None)
        assert st == want, f"{name}: status {st} ({_err()})"


def test_resample_refusals():
    lib = _cabi().lib
    good = dict(i=P, o=P, planes=2, oh=4, ow=4, sy=P, sx=P, dtype=1)
    cases = [("in", dict(i=None), INVALID), ("out", dict(o=None), INVALID), ("src_y", dict(sy=None), INVALID),
             ("src_x", dict(sx=None), INVALID), ("planes 0", dict(planes=0), INVALID), ("oh 0", dict(oh=0), INVALID),
             ("ow 0", dict(ow=0), INVALID), ("dtype 3", dict(dtype=3), INVALID), ("65536 planes", dict(planes=65536), UNSUPPORTED)]
    for name, over, want in cases:
        a = {**good, **over}
        st = lib.td_resample_nearest(a["i"], a["o"], a["planes"], 8, 8, a["oh"], a["ow"], a["sy"], a["sx"], a["dtype"], None)
        assert st == want, f"{name}: status {st} ({_err()})"


def test_affine_clamp_refusals():
    lib = _cabi().lib
    names = ["x", "mean_new", "std_new", "mean_old", "std_old", "lo", "hi"]
    for i, name in enumerate(names):
        ptrs = [P] * 7
        ptrs[i] = None
        st = lib.td_affine_clamp(ptrs[0], 1, 3, 16, 2, *ptrs[1:], None)
        assert st == INVALID, f"{name}: status {st} ({_err()})"
    for name, (B, C, HW, dt), want in [("B 0", (0, 3, 16, 2), INVALID), ("C 0", (1, 0, 16, 2), INVALID), ("HW 0", (1, 3, 0, 2), INVALID),
                                       ("B*C = 65536", (2, 32768, 16, 2), UNSUPPORTED), ("dtype 3", (1, 3, 16, 3), INVALID)]:
        st = lib.td_affine_clamp(P, B, C, HW, dt, P, P, P, P, P, P, None)
        assert st == want, f"{name}: status {st} ({_err()})"


# ---------------------------------------------------------------------------------------------------------------------
# 1. td_gn_stats
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_gn_stats_every_form_against_float64(dn):
    """<T, VECTOR, MINMAX>: vector with and without min / max, scalar because seg_len % v != 0 and scalar because x is
    one element off 16-byte alignment (the scalar path always tracks min / max); biased and unbiased."""
    dt = DTS[dn]
    T, vec = TNAME[dt], 16 // ES[dt]
    nseg, seg_len = 6, 37 * 1024
    base = _randn((nseg * seg_len + 1,), 10, 1.7, 0.6).to(dt)
    cases = [("vector + min/max", base[:nseg * seg_len], nseg, seg_len, True, True, (T, "true", "true")),
             ("vector", base[:nseg * seg_len], nseg, seg_len, False, True, (T, "true", "false")),
             ("scalar: seg_len % v", base[:nseg * (seg_len - 1)], nseg, seg_len - 1, False, True, (T, "false", "true")),
             ("scalar: unaligned x", base[1:], nseg, seg_len, True, False, (T, "false", "true"))]
    for name, x, ns, sl, mm, aligned, want in cases:
        assert (x.data_ptr() % 16 == 0) == aligned and (sl % vec == 0) == (name != "scalar: seg_len % v")
        for unbiased in (False, True):
            forms = _check_stats(x, ns, sl, unbiased, f"{dn} {name} unbiased={unbiased}", minmax=mm, aligned=aligned)
            assert forms == {want}, f"{dn} {name}: launched {sorted(forms)}"


# (nseg, seg_len) per dtype: every branch of the plan on the device
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_gn_stats_plan_branches_against_float64(dn):
    """One chunk, the seg_len / (256 v)-limited and the want-limited counts, the chunk-size-limited count, a partial
    last chunk, and the 1024-chunk cap (more than 2^24 fp32 / 2^25 16-bit elements in one segment)."""
    dt = DTS[dn]
    es = ES[dt]
    vec = 16 // es
    cap = 1024 * (65536 // es) + vec
    for i, (nseg, seg_len) in enumerate([(1, 1000), (1, 5000), (2, 1_000_000), (64, 300_000), (1, cap), (1, cap - 1)]):
        chunk, chunks, _ = plan_stats(nseg, seg_len, es)
        x = _randn((nseg * seg_len,), 20 + i, 2.0, -0.3).to(dt)
        _check_stats(x, nseg, seg_len, i % 2 == 1, f"{dn} plan {nseg}x{seg_len} ({chunks} chunks of {chunk})")
        if seg_len >= cap - 1:
            assert chunks == 1024
        del x
    torch.cuda.empty_cache()


PROBE = {torch.float16: (2.0 ** -10, 1.0, 1 << 17), torch.bfloat16: (2.0 ** -10, 2.0 ** -3, 1 << 15),
         torch.float32: (2.0 ** -20, 8.0, 1 << 20)}


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("form", ["vector", "scalar"])
def test_gn_stats_coverage_probes(dn, form):
    """Constant segments of c with one element c + delta (delta a power of two): mean - c = delta / n and
    var = delta^2 (n - 1) / n^2 (biased) or delta^2 / n (unbiased) to 1e-3, min / max exact.  The probe sits on the
    first element of a chunk (the shift k), the last element of a chunk, the scalar tail past the last full vector,
    the last element of the segment, and the first element of the next segment (bleed between segments)."""
    dt = DTS[dn]
    c, delta, n = PROBE[dt]
    vec = 16 // ES[dt]
    if form == "scalar":
        n += vec - 1
    nseg = 5
    chunk, chunks, vector = plan_stats(nseg, n, ES[dt])
    assert vector == (form == "vector") and chunks >= 3
    tail = n - 1 - (n % vec) + 1 if form == "scalar" else n - vec
    pos = [chunk, 2 * chunk - 1, tail, n - 1, 0]
    x = torch.full((nseg, n), c, dtype=dt, device="cuda")
    for s, p in enumerate(pos):
        x[s, p] = c + delta
    assert float(x[0, chunk]) == c + delta
    for unbiased, mm in [(True, True), (False, False)]:
        out = _tv()._segment_stats(x, nseg, n, unbiased=unbiased, want_minmax=mm)
        var, mean = out[0].double().cpu(), out[1].double().cpu()
        want_v = delta * delta / n if unbiased else delta * delta * (n - 1) / (n * n)
        for s, p in enumerate(pos):
            rm = abs((mean[s].item() - c) / (delta / n) - 1)
            rv = abs(var[s].item() / want_v - 1)
            assert rm <= 1e-3 and rv <= 1e-3, f"{dn} {form} probe at {p} (chunk {chunk}): mean err {rm:.3g}, var err {rv:.3g}"
        if mm:
            assert (out[2] == c).all() and (out[3] == c + delta).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_gn_stats_values(dn):
    """Constant segments (var exactly 0, mean exactly c), mean >> std, +-0, fp16 subnormals, magnitudes near the
    format's maximum (fp16: +-65504 with full spread, d^2 ~ 1.7e10; bf16: a constant segment at the maximum and a spread
    at 2^40, where n d^2 stays finite)."""
    dt = DTS[dn]
    tv = _tv()
    for c in (1.75, -3.0, 2.0 ** -14, float(torch.finfo(dt).max)):
        x = torch.full((4, 9000), c, dtype=dt, device="cuda")
        for unbiased in (False, True):
            var, mean, lo, hi = tv._segment_stats(x, 4, 9000, unbiased=unbiased, want_minmax=True)
            assert (var == 0).all() and (mean == float(x[0, 0])).all() and (lo == float(x[0, 0])).all() and (hi == float(x[0, 0])).all()
    _check_stats(_randn((3 * 20000,), 30, 0.01, 100.0).to(dt), 3, 20000, False, f"{dn} mean >> std")
    z = torch.zeros(4 * 4096, dtype=dt, device="cuda")
    z[1::3] = -0.0
    var, mean, lo, hi = tv._segment_stats(z, 4, 4096, unbiased=True, want_minmax=True)
    assert (var == 0).all() and (mean == 0).all() and (lo == 0).all() and (hi == 0).all()
    if dt == torch.float16:
        sub = (_randn((2 * 8192,), 31, 2.0 ** -18)).to(dt)
        assert ((sub != 0) & (sub.abs() < 2.0 ** -14)).sum() > 8000
        _check_stats(sub, 2, 8192, True, "fp16 subnormals")
        big = (_randn((2 * 8192,), 32, 30000.0)).clamp(-65504, 65504).to(dt)
        big[::1000] = 65504.0
        big[1::1000] = -65504.0
        _check_stats(big, 2, 8192, False, "fp16 near +-65504")
    if dt == torch.bfloat16:
        _check_stats((_randn((2 * 8192,), 33, 2.0 ** 40)).to(dt), 2, 8192, True, "bf16 at 2^40")
    if dt == torch.float32:
        _check_stats((_randn((2 * 8192,), 34, 2.0 ** 50)), 2, 8192, True, "fp32 at 2^50")


@pytest.mark.gpu
def test_gn_stats_limits():
    """65535 segments work (one chunk each); a workspace of exactly the planned size works."""
    tv = _tv()
    lib = _cabi().lib
    x = _randn((65535 * 8,), 40, 1.0, 0.5).to(torch.float16)
    var, mean = tv._segment_stats(x, 65535, 8, unbiased=False)
    mu, v64, *_ , e_mean, e_var = _stats64(x, 65535, 8, False)
    assert ((mean.double() - mu).abs() <= e_mean).all() and ((var.double() - v64).abs() <= e_var).all()
    for nseg, seg_len, dt in [(65535, 8, torch.float16), (3, 50_000, torch.float32), (1, 5000, torch.bfloat16)]:
        x = _randn((nseg * seg_len,), 41, 1.0).to(dt)
        need = workspace_bytes(nseg, seg_len, ES[dt])
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        mean = torch.empty(nseg, device="cuda")
        var = torch.empty(nseg, device="cuda")
        assert lib.td_gn_stats(x.data_ptr(), nseg, seg_len, CODE[dt], 0, ws.data_ptr(), need, mean.data_ptr(), var.data_ptr(), None,
                               None, _stream()) == OK, _err()
        assert lib.td_gn_stats(x.data_ptr(), nseg, seg_len, CODE[dt], 0, ws.data_ptr(), need - 1, mean.data_ptr(), var.data_ptr(),
                               None, None, _stream()) == CAPACITY
        mu, v64, *_, e_mean, e_var = _stats64(x, nseg, seg_len, False)
        assert ((mean.double() - mu).abs() <= e_mean).all() and ((var.double() - v64).abs() <= e_var).all()


# ---------------------------------------------------------------------------------------------------------------------
# 2. td_gn_apply
# ---------------------------------------------------------------------------------------------------------------------
def _apply_call(x, y, B, C, HW, groups, mean, var, per_batch, gamma, beta, act):
    lib = _cabi().lib
    return lib.td_gn_apply(x.data_ptr(), y.data_ptr(), B, C, HW, CODE[x.dtype], groups, mean.data_ptr(), var.data_ptr(), int(per_batch),
                           gamma.data_ptr() if gamma is not None else None, beta.data_ptr() if beta is not None else None, 1e-6,
                           int(act), _stream())


def _apply_case(dt, B, C, HW, groups, per_batch, has_g, has_b, act, seed, x_off=0, y_off=0, inplace=False, xscale=2.0):
    """Run td_gn_apply on x [B, C, HW] stored `x_off` elements into its buffer (y `y_off`), check it against float64
    and return the launched forms."""
    buf = _randn((B * C * HW + 8,), seed, xscale, 0.3).to(dt)
    x = buf[x_off:x_off + B * C * HW]
    xin = x.clone()
    if inplace:
        y = x
    else:
        ybuf = torch.full((B * C * HW + 8,), float("nan"), dtype=dt, device="cuda")
        y = ybuf[y_off:y_off + B * C * HW]
    ns = B * groups if per_batch else groups
    mean = _randn((ns,), seed + 1, 0.4, 0.2)
    var = _randn((ns,), seed + 2, 0.5).abs() + 0.3
    gamma = _randn((C,), seed + 3, 0.5, 1.0) if has_g else None
    beta = _randn((C,), seed + 4, 0.3) if has_b else None
    box = {}

    def run():
        if inplace:
            x.copy_(xin)
        box["st"] = _apply_call(x, y, B, C, HW, groups, mean, var, per_batch, gamma, beta, act)
    forms = _forms(run, K_APPLY)
    assert box["st"] == OK, _err()
    ref, bound = _apply64(xin.view(B, C, HW), mean, var, gamma, beta, act, groups, per_batch)
    _within(y.view(B, C, HW), ref, bound, "gn_apply", dt,
            f"{_dn(dt)} B={B} C={C} HW={HW} per_batch={per_batch} g={has_g} b={has_b} act={act} x_off={x_off} y_off={y_off} inplace={inplace}")
    return forms


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_gn_apply_every_form_against_float64(dn):
    """Vector and scalar forms (HW % v != 0, x unaligned, y unaligned), in place in both, per-batch statistics on and
    off with B = 3, gamma / beta each absent, SiLU on and off (inputs reach t < -87)."""
    dt = DTS[dn]
    T, vec = TNAME[dt], 16 // ES[dt]
    B, C, groups = 3, 64, 32
    HW = 40 * vec
    vector, scalar = {(T, "true")}, {(T, "false")}
    seed = 100
    for per_batch in (False, True):
        for has_g, has_b, act in [(True, True, True), (True, True, False), (False, True, True), (True, False, False), (False, False, True)]:
            seed += 10
            assert _apply_case(dt, B, C, HW, groups, per_batch, has_g, has_b, act, seed) == vector
            assert _apply_case(dt, B, C, HW + 1, groups, per_batch, has_g, has_b, act, seed + 5) == scalar
    for kw, want in [(dict(x_off=1), scalar), (dict(y_off=1), scalar), (dict(inplace=True), vector), (dict(inplace=True, x_off=1), scalar)]:
        seed += 10
        assert _apply_case(dt, B, C, HW, groups, True, True, True, True, seed, **kw) == want, kw
    # SiLU far into the negative range: |x| ~ 200 sigma drives t below -87 (the __fdividef zero)
    assert _apply_case(dt, 1, 32, HW, 32, False, True, True, True, 190, xscale=150.0) == vector


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_gn_apply_grid_and_plane_limits(dn):
    """grid.x capped at 4096 CTAs: one plane of more than 4096 * 1024 * v elements (vector) / 4096 * 1024 (scalar) makes
    every thread loop; B * C = 65535 planes work."""
    dt = DTS[dn]
    T, vec = TNAME[dt], 16 // ES[dt]
    for HW, want in [(4096 * 1024 * vec + 4 * vec, (T, "true")), (4096 * 1024 + 3, (T, "false"))]:
        x = _randn((HW,), 200, 1.5, 0.2).to(dt)
        y = torch.empty_like(x)
        mean, var = torch.tensor([0.25], device="cuda"), torch.tensor([1.7], device="cuda")
        gamma, beta = torch.tensor([1.3], device="cuda"), torch.tensor([-0.4], device="cuda")
        forms = _forms(lambda: _apply_call(x, y, 1, 1, HW, 1, mean, var, False, gamma, beta, True), K_APPLY)
        assert forms == {want}
        step = 1 << 22
        for s in range(0, HW, step):
            xs = x[s:s + step].view(1, 1, -1)
            ref, bound = _apply64(xs, mean, var, gamma, beta, True, 1, False)
            _within(y[s:s + step].view(1, 1, -1), ref, bound, "gn_apply", dt, f"{dn} HW={HW} from {s}")
        del x, y
    torch.cuda.empty_cache()
    C, groups = 65535, 5
    x = _randn((C * 8,), 201, 1.0).to(dt).view(1, C, 8)
    y = torch.empty_like(x)
    mean, var = _randn((groups,), 202, 0.3), _randn((groups,), 203).abs() + 0.5
    assert _apply_call(x, y, 1, C, 8, groups, mean, var, False, None, None, False) == OK, _err()
    ref, bound = _apply64(x, mean, var, None, None, False, groups, False)
    _within(y, ref, bound, "gn_apply", dt, f"{dn} B*C = 65535")


# ---------------------------------------------------------------------------------------------------------------------
# 3. td_copy_region / td_resample_nearest: bit-exact
# ---------------------------------------------------------------------------------------------------------------------
def _copy_case(dt, planes, rows, cols, sp, spitch, dp, dpitch, s_off=0, d_off=0, seed=0):
    """Copy a [planes, rows, cols] region between two flat buffers of random bit patterns (dst pre-filled with a
    sentinel); everything outside the region must keep its sentinel.  Returns the launched forms."""
    lib = _cabi().lib
    n_src = s_off + (planes - 1) * sp + (rows - 1) * spitch + cols
    n_dst = d_off + (planes - 1) * dp + (rows - 1) * dpitch + cols
    src = _bits(n_src + 8, dt, seed)
    sentinel = torch.full((n_dst + 8,), 0x5a5a5a5a if dt == torch.float32 else 0x5a5a, dtype=INT[dt], device="cuda").view(dt)
    dst = sentinel.clone()

    def run():
        assert lib.td_copy_region(src.data_ptr() + s_off * ES[dt], dst.data_ptr() + d_off * ES[dt], planes, rows, cols, sp, spitch, dp,
                                  dpitch, CODE[dt], _stream()) == OK, _err()
    forms = _forms(run, K_COPY)
    want = sentinel.clone()
    want.view(INT[dt]).as_strided((planes, rows, cols), (dp, dpitch, 1), d_off).copy_(
        src.view(INT[dt]).as_strided((planes, rows, cols), (sp, spitch, 1), s_off))
    assert torch.equal(dst.view(INT[dt]), want.view(INT[dt])), f"{_dn(dt)} copy {planes}x{rows}x{cols} differs"
    return forms


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_copy_region_vector_conditions_bit_exact(dn):
    """The vector form needs all seven conditions; each one broken on its own falls back to the scalar form."""
    dt = DTS[dn]
    v = 16 // ES[dt]
    W = WORD[dt]
    planes, rows, cols = 3, 17, 6 * v
    sp, spitch, dp, dpitch = 20 * 8 * v, 8 * v, 24 * 9 * v, 9 * v
    assert _copy_case(dt, planes, rows, cols, sp, spitch, dp, dpitch, seed=1) == {(W, "true")}
    broken = [dict(s_off=1), dict(d_off=1), dict(cols=cols - 1), dict(spitch=spitch + 1), dict(dpitch=dpitch + 1), dict(sp=sp + 1),
              dict(dp=dp + 1)]
    for i, over in enumerate(broken):
        a = dict(planes=planes, rows=rows, cols=cols, sp=sp, spitch=spitch, dp=dp, dpitch=dpitch, s_off=0, d_off=0)
        a.update(over)
        assert _copy_case(dt, seed=2 + i, **a) == {(W, "false")}, over


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_copy_region_grid_loops_and_sizes(dn):
    """rows > 65535 (capped grid.y), cols above 64 * 256 * v (vector) / 64 * 256 (scalar) (capped grid.x), 65535 planes,
    and zero-size copies that write nothing."""
    dt = DTS[dn]
    v = 16 // ES[dt]
    W = WORD[dt]
    rows = 65535 + 9
    assert _copy_case(dt, 1, rows, 2 * v, 0, 3 * v, 0, 4 * v, seed=20) == {(W, "true")}
    assert _copy_case(dt, 1, rows, 3, 0, 5, 0, 7, seed=21) == {(W, "false")}
    cv = 64 * 256 * v * 2 + v
    assert _copy_case(dt, 2, 3, cv, 3 * cv, cv, 4 * (cv + v), cv + v, seed=22) == {(W, "true")}
    cs = 64 * 256 * 2 + 1
    assert _copy_case(dt, 2, 3, cs, 3 * cs, cs, 3 * cs + 1, cs, seed=23) == {(W, "false")}
    assert _copy_case(dt, 65535, 1, v, v, v, 2 * v, v, seed=24) == {(W, "true")}
    lib = _cabi().lib
    src, dst = _bits(64, dt, 25), _bits(64, dt, 26)
    before = dst.clone()
    for p, r, c in [(0, 2, 2), (2, 0, 2), (2, 2, 0)]:
        assert lib.td_copy_region(src.data_ptr(), dst.data_ptr(), p, r, c, 8, 4, 8, 4, CODE[dt], _stream()) == OK
    torch.cuda.synchronize()
    assert torch.equal(dst.view(INT[dt]), before.view(INT[dt]))


def _resample_case(dt, planes, H, W, sy, sx, seed):
    lib = _cabi().lib
    x = _bits(planes * H * W, dt, seed).view(planes, H, W)
    sy_d = torch.as_tensor(sy, dtype=torch.int32, device="cuda")
    sx_d = torch.as_tensor(sx, dtype=torch.int32, device="cuda")
    oh, ow = len(sy), len(sx)
    out = torch.full((planes * oh * ow + 8,), 0x5a5a5a5a if dt == torch.float32 else 0x5a5a, dtype=INT[dt], device="cuda").view(dt)
    before = out.clone()

    def run():
        assert lib.td_resample_nearest(x.data_ptr(), out.data_ptr(), planes, H, W, oh, ow, sy_d.data_ptr(), sx_d.data_ptr(), CODE[dt],
                                       _stream()) == OK, _err()
    forms = _forms(run, K_RESAMPLE)
    xi = x.view(INT[dt])
    want = xi[:, sy_d.long()][:, :, sx_d.long()].reshape(-1)
    assert torch.equal(out.view(INT[dt])[:planes * oh * ow], want), f"{_dn(dt)} resample {planes}x{H}x{W} -> {oh}x{ow}"
    assert torch.equal(out.view(INT[dt])[planes * oh * ow:], before.view(INT[dt])[planes * oh * ow:])
    return forms


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_resample_nearest_bit_exact(dn):
    """in[:, sy][:, :, sx] with nearest_exact_indices at the estimator scales of the census shapes, B = 1..3; oh > 65535
    and ow > 64 * 256 (the capped grid loops); 65535 planes."""
    dt = DTS[dn]
    tv = _tv()
    want = {(WORD[dt],)}
    for B, C, H, W, tile in [(1, 4, 40, 52, 16), (3, 4, 40, 52, 16), (2, 3, 200, 264, 64), (1, 3, 136, 200, 64), (2, 4, 70, 100, 32)]:
        s = tile / max(H, W)
        _, sy = tv.nearest_exact_indices(H, s)
        _, sx = tv.nearest_exact_indices(W, s)
        assert _resample_case(dt, B * C, H, W, sy, sx, 300 + H) == want
    g = torch.Generator().manual_seed(301)
    assert _resample_case(dt, 1, 70000, 3, torch.randint(0, 70000, (65535 + 20,), generator=g), [2, 0, 1, 1], 302) == want
    assert _resample_case(dt, 2, 3, 40000, [1, 2], torch.randint(0, 40000, (64 * 256 * 2 + 5,), generator=g), 303) == want
    assert _resample_case(dt, 65535, 2, 2, [1], [0, 1], 304) == want


# ---------------------------------------------------------------------------------------------------------------------
# 4. td_affine_clamp: bit-exact against eager torch on the same device
# ---------------------------------------------------------------------------------------------------------------------
def _clamp_case(dt, x, mn, sn, mo, so, lo, hi, what):
    """x [B, C, HW] (dtype); statistics [C] and bounds (scalars) are made dtype tensors on the device, as the reference
    makes them (torch.std_mean(..., keepdim=True), z.min() / z.max()); the kernel takes their fp32 values."""
    lib = _cabi().lib
    B, C, HW = x.shape
    st = [torch.tensor(v, device="cuda").to(dt) for v in (mn, sn, mo, so)]
    lo_t, hi_t = (torch.tensor(float(v), device="cuda").to(dt) for v in (lo, hi))
    want = ((x - st[0].view(1, C, 1)) / st[1].view(1, C, 1) * st[3].view(1, C, 1) + st[2].view(1, C, 1)).clamp_(lo_t, hi_t)
    got = x.clone()
    f32 = [t.float().contiguous() for t in st] + [lo_t.float().view(1), hi_t.float().view(1)]
    box = {}

    def run():
        got.copy_(x)
        box["st"] = lib.td_affine_clamp(got.data_ptr(), B, C, HW, CODE[dt], *(t.data_ptr() for t in f32), _stream())
    forms = _forms(run, K_CLAMP)
    assert box["st"] == OK, _err()
    assert forms == {(TNAME[dt],)}, forms
    assert_bit_equal(got, want, f"{_dn(dt)} {what}")


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_affine_clamp_matches_eager_torch_bit_for_bit(dn):
    dt = DTS[dn]
    inf, nan = float("inf"), float("nan")
    B, C, HW = 2, 3, 1000
    x = _randn((B, C, HW), 400, 2.0, 0.1).to(dt)
    stats = ([0.1, -0.3, 0.7], [1.3, 0.6, 2.1], [0.2, 0.05, -0.4], [0.9, 1.7, 0.4])
    _clamp_case(dt, x, *stats, -1.5, 1.25, "ordinary")
    _clamp_case(dt, x, *stats, -inf, inf, "lo / hi = -+inf (DemoFusion)")
    # x exactly at the bounds and -0.0 against a bound of 0 (identity transform)
    ident = ([0.0] * C, [1.0] * C, [1.0] * C, [0.0] * C)
    xb = torch.tensor([-1.5, 1.25, -0.0, 0.0, -1.5000001, 1.2500001, 0.5, -0.7], device="cuda").to(dt).repeat(B, C, 16)
    _clamp_case(dt, xb, *ident, -1.5, 1.25, "x at the bounds")
    _clamp_case(dt, xb, *ident, 0.0, 1.25, "-0.0 against lo = 0")
    _clamp_case(dt, xb, *ident, -1.5, 0.0, "-0.0 against hi = 0")
    _clamp_case(dt, xb, *ident, 0.0, 0.0, "lo = hi = 0")
    # NaN and +-inf in x
    xn = x.clone()
    xn[:, :, ::7] = nan
    xn[:, :, 1::7] = inf
    xn[:, :, 2::7] = -inf
    _clamp_case(dt, xn, *stats, -1.5, 1.25, "NaN / inf in x")
    _clamp_case(dt, xn, *stats, -inf, inf, "NaN / inf in x, infinite bounds")
    # sn = 0: 0 / 0 where x == mn, +-x / 0 elsewhere
    xz = x.clone()
    xz[:, :, ::3] = torch.tensor([0.1, -0.3, 0.7], device="cuda").to(dt).view(1, C, 1)
    zero = (stats[0], [0.0, 1.0, 0.0], stats[2], stats[3])
    _clamp_case(dt, xz, *zero, -1.5, 1.25, "sn = 0")
    _clamp_case(dt, xz, *zero, -inf, inf, "sn = 0, infinite bounds")
    # NaN bounds
    _clamp_case(dt, x, *stats, nan, 1.25, "lo = NaN")
    _clamp_case(dt, x, *stats, -1.5, nan, "hi = NaN")
    _clamp_case(dt, x, *stats, nan, nan, "lo = hi = NaN")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the fast-mode path end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("flat", [False, True], ids=["random", "flat_channel"])
def test_fast_mode_estimator_input_batched(dn, B, flat):
    """B > 1 merges the per-(b, c) moments in Python.  Tolerances of test_gpu_vae.py (f32 2e-5, f16 3e-2; bf16: 8 x the
    fp16 one); the NaN masks must be identical (a channel constant over the whole batch has std_new = 0: 0 / 0)."""
    from oracle import vae
    dt = DTS[dn]
    g = torch.Generator().manual_seed(500 + B)
    z = (torch.randn((B, 4, 70, 100), generator=g) * 5 + 1).to(dt)
    if flat:     # in fp32, the mean of three copies of either value is not the value itself
        z[:, 1] = 0.79549014
        z[:, 2] = 0.39662069
    want = vae.fast_mode_estimator_input(z.float() if dt == torch.float32 else z, 32)
    got = _tv().fast_mode_estimator_input(z.cuda(), 32).cpu()
    assert got.shape == want.shape and got.dtype == dt
    nan_g, nan_w = got.float().isnan(), want.float().isnan()
    assert torch.equal(nan_g, nan_w), f"NaN masks differ: {int(nan_g.sum())} vs {int(nan_w.sum())}"
    assert nan_w.any() == flat
    tol = {"f32": 2e-5, "f16": 3e-2, "bf16": 0.24}[dn]
    ok = ~nan_w
    assert (got.float()[ok] - want.float()[ok]).abs().max() <= tol * max(1.0, want.float()[ok].abs().max().item())


def _flat_inputs(is_dec, H, W, tile):
    tv = _tv()
    from oracle import synth
    if is_dec:
        z = synth.latent(5, (1, 4, H, W), torch.float32)
        z[:, 1] = 0.4375
        return [("latent with one constant channel", z)]
    flat = torch.tensor([0.7, -0.2, 0.4]).view(1, 3, 1, 1).expand(1, 3, H, W).contiguous()
    s = tile / max(H, W)
    _, sy = tv.nearest_exact_indices(H, s)
    y = next(i for i in range(H) if i not in set(sy.tolist()))
    detail = flat.clone()
    detail[:, :, y, W // 2] = 0.2
    return [("flat colour", flat), ("flat with a sub-stride detail", detail)]


def _spy_estimate(monkeypatch):
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    seen = []
    real = ve.Executor.estimate

    def est(self, act, color_fix):
        r = real(self, act, color_fix)
        seen.append(r)
        return r
    monkeypatch.setattr(ve.Executor, "estimate", est)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("is_dec", [True, False], ids=["decoder", "encoder"])
def test_vaehook_fast_mode_on_flat_inputs_falls_back_like_the_reference(monkeypatch, is_dec):
    """A constant channel in the estimator's input makes its re-standardisation 0 / 0.  The reference then disables fast
    mode and runs slow mode; so must VAEHook (Executor.estimate returns False), on the module backend (small fp32 nets)
    and on the tensor-core backend (SD-width fp16 nets)."""
    from oracle import vae
    from oracle.make_golden import vae_case_inputs
    from test_gpu_vae import _sd_width_net
    tv = _tv()
    # fp32 convolutions in fp32 on both sides, as in test_gpu_vae.py (slow mode on flat tiles divides by sqrt(var + eps)
    # with var ~ 0, which magnifies TF32 rounding)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    H, W, tile = (40, 52, 16) if is_dec else (200, 264, 64)
    seen = _spy_estimate(monkeypatch)
    for name, z in _flat_inputs(is_dec, H, W, tile):
        net, _ = vae_case_inputs(is_dec, H, W)
        with torch.no_grad():
            want = vae.vae_hook_call(net, z, tile, is_dec, True, False)
        net_gpu, _ = vae_case_inputs(is_dec, H, W)
        net_gpu = net_gpu.cuda()
        hook = tv.VAEHook(net_gpu, tile, is_dec, fast_decoder=True, fast_encoder=True, color_fix=False)
        seen.clear()
        with torch.no_grad():
            got = hook(z.cuda())
        assert hook.backend_name == "modules" and seen == [False], f"{name}: estimate returned {seen}"
        scale = max(1.0, want.abs().max().item())
        err = (got.cpu() - want).abs().max().item()
        assert err <= 3e-4 * scale, f"{name} (fp32 modules): max err {err} vs scale {scale}"

        ref_net = _sd_width_net(is_dec, 3 if is_dec else 4).cuda()
        with torch.no_grad():
            want = vae.vae_hook_call(ref_net, z.cuda(), tile, is_dec, True, False).cpu()
        net16 = _sd_width_net(is_dec, 3 if is_dec else 4).cuda().half()
        hook = tv.VAEHook(net16, tile, is_dec, fast_decoder=True, fast_encoder=True, color_fix=False)
        seen.clear()
        with torch.no_grad():
            got = hook(z.cuda().half())
        assert hook.backend_name == "wgmma" and seen == [False], f"{name}: estimate returned {seen}"
        diff = (got.cpu().float() - want).abs()
        scale = want.abs().max().item()
        assert diff.mean().item() <= 2e-3 * scale and diff.max().item() <= 3e-2 * scale, (name, diff.mean().item() / scale,
                                                                                         diff.max().item() / scale)
        del ref_net, net16


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_demofusion_renormalise_of_a_constant_is_nan(dn):
    """(g - g.mean()) / g.std() * x.std() + x.mean() with a constant g is 0 / 0 everywhere: NaN, as in the reference
    (which has no clamp there)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    dt = DTS[dn]
    g_ = torch.full((2, 4, 24, 32), 0.375, dtype=dt, device="cuda")
    x = _randn((2, 4, 24, 32), 600, 1.2, 0.3).to(dt)
    want = (g_.float() - g_.float().mean()) / g_.float().std() * x.float().std() + x.float().mean()
    assert want.isnan().all()
    got = DemoFusion._renormalise(None, g_.clone(), x)
    assert got.isnan().all(), f"{int((~got.isnan()).sum())} elements are not NaN (e.g. {got.flatten()[0].item()})"


# ---------------------------------------------------------------------------------------------------------------------
# 6. census: every (kernel, shape, dtype, options) the module backend issues, replayed against float64
# ---------------------------------------------------------------------------------------------------------------------
CENSUS_RUNS = [(True, 40, 52, 16), (False, 200, 264, 64)]
DNAME = {0: "f16", 1: "bf16", 2: "f32"}


class _LibSpy:
    """Stands in for tilevae's handle of the library and records the td_gn_stats / td_gn_apply signatures."""

    def __init__(self, real, seen):
        self._real, self._seen = real, seen

    def __getattr__(self, name):
        f = getattr(self._real, name)
        if name == "td_gn_stats":
            def stats(x, nseg, seg_len, dtype, unbiased, *rest):
                self._seen.add(("stats", int(nseg), int(seg_len), DNAME[dtype], bool(unbiased), rest[4] is not None))
                return f(x, nseg, seg_len, dtype, unbiased, *rest)
            return stats
        if name == "td_gn_apply":
            def apply(x, y, B, C, HW, dtype, groups, mean, var, per_batch, gamma, beta, eps, act, stream):
                self._seen.add(("apply", int(B), int(C), int(HW), DNAME[dtype], int(groups), bool(per_batch), gamma is not None,
                                beta is not None, bool(act)))
                return f(x, y, B, C, HW, dtype, groups, mean, var, per_batch, gamma, beta, eps, act, stream)
            return apply
        return f


def record_census():
    """Distinct td_gn_stats / td_gn_apply signatures of the module backend: SD-width encoder and decoder, fast and slow
    mode, wrap on and off, fp32 and (with pick_backend forced to the module backend) fp16 / bf16."""
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    from oracle import synth
    from test_gpu_vae import _sd_width_net
    tv = _tv()
    seen = set()
    real_lib, real_pick = tv.lib, ve.pick_backend
    try:
        tv.lib = _LibSpy(real_lib, seen)
        ve.pick_backend = lambda program, device, dtype: ve.ModuleBackend(program, device, dtype)
        for is_dec, H, W, tile in CENSUS_RUNS:
            base = _sd_width_net(is_dec, 3 if is_dec else 4)
            for dt in DTS.values():
                net = copy.deepcopy(base).cuda().to(dt)
                z = synth.latent(5 if is_dec else 6, (1, 4 if is_dec else 3, H, W), dt).cuda()
                for fast in (True, False):
                    for wrap in (False, True):
                        hook = tv.VAEHook(net, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
                        hook.wrap_x = hook.wrap_y = wrap
                        with torch.no_grad():
                            hook(z)
                        assert hook.backend_name == "modules"
                del net
    finally:
        tv.lib, ve.pick_backend = real_lib, real_pick
    return sorted(seen, key=repr)


# recorded by record_census() on an H100 (SD-width encoder / decoder, fast and slow mode, wrap on and off, three dtypes)
CENSUS = [
    ('apply', 1, 128, 12288, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 12288, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 12288, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 12544, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 12544, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 12544, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 1296, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 1296, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 1296, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 13440, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 13440, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 13440, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 14400, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 14400, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 14400, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 16384, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 16384, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 16384, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 2304, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 2304, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 2304, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 3072, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 3072, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 3072, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 3136, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 3136, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 3136, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 3360, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 3360, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 3360, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 3600, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 3600, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 3600, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 4096, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 4096, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 4096, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 5184, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 5184, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 5184, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 55296, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 55296, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 55296, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 58368, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 58368, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 58368, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 768, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 768, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 768, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 78400, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 78400, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 78400, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 80640, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 80640, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 80640, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 87552, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 87552, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 87552, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 9216, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 9216, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 9216, 'f32', 32, False, True, True, True),
    ('apply', 1, 128, 92416, 'bf16', 32, False, True, True, True),
    ('apply', 1, 128, 92416, 'f16', 32, False, True, True, True),
    ('apply', 1, 128, 92416, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 1024, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 1024, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 1024, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 12288, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 12288, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 12288, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 1296, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 1296, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 1296, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 13824, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 13824, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 13824, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 14592, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 14592, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 14592, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 192, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 192, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 192, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 19600, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 19600, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 19600, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 20160, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 20160, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 20160, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 21888, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 21888, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 21888, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 2304, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 2304, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 2304, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 23104, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 23104, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 23104, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 3072, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 3072, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 3072, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 3136, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 3136, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 3136, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 324, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 324, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 324, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 3360, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 3360, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 3360, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 3600, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 3600, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 3600, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 4096, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 4096, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 4096, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 55296, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 55296, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 55296, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 576, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 576, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 576, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 58368, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 58368, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 58368, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 768, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 768, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 768, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 784, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 784, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 784, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 78400, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 78400, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 78400, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 80640, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 80640, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 80640, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 840, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 840, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 840, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 87552, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 87552, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 87552, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 900, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 900, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 900, 'f32', 32, False, True, True, True),
    ('apply', 1, 256, 92416, 'bf16', 32, False, True, True, True),
    ('apply', 1, 256, 92416, 'f16', 32, False, True, True, True),
    ('apply', 1, 256, 92416, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 1024, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 1024, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 1024, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 1225, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 1225, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 1225, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 1225, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 1225, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 1225, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 1260, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 1260, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 1260, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 1260, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 1260, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 1260, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 1368, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 1368, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 1368, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 1368, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 1368, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 1368, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 13824, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 13824, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 13824, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 144, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 144, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 144, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 144, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 144, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 144, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 1444, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 1444, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 1444, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 1444, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 1444, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 1444, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 14592, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 14592, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 14592, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 192, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 192, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 192, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 192, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 192, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 192, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 196, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 196, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 196, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 196, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 196, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 196, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 19600, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 19600, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 19600, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 20160, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 20160, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 20160, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 210, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 210, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 210, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 210, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 210, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 210, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 21888, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 21888, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 21888, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 225, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 225, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 225, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 225, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 225, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 225, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 23104, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 23104, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 23104, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 256, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 256, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 256, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 256, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 256, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 256, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 3072, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 3072, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 3072, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 324, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 324, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 324, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 3456, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 3456, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 3456, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 3648, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 3648, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 3648, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 48, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 48, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 48, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 48, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 48, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 48, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 4900, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 4900, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 4900, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 5040, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 5040, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 5040, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 5472, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 5472, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 5472, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 576, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 576, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 576, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 5776, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 5776, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 5776, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 768, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 768, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 768, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 784, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 784, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 784, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 81, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 81, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 81, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 81, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 81, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 81, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 840, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 840, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 840, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 864, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 864, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 864, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 864, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 864, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 864, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 900, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 900, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 900, 'f32', 32, False, True, True, True),
    ('apply', 1, 512, 912, 'bf16', 32, False, True, True, False),
    ('apply', 1, 512, 912, 'bf16', 32, False, True, True, True),
    ('apply', 1, 512, 912, 'f16', 32, False, True, True, False),
    ('apply', 1, 512, 912, 'f16', 32, False, True, True, True),
    ('apply', 1, 512, 912, 'f32', 32, False, True, True, False),
    ('apply', 1, 512, 912, 'f32', 32, False, True, True, True),
    ('stats', 3, 3072, 'bf16', True, False),
    ('stats', 3, 3072, 'f16', True, False),
    ('stats', 3, 3072, 'f32', True, False),
    ('stats', 3, 52800, 'bf16', True, True),
    ('stats', 3, 52800, 'f16', True, True),
    ('stats', 3, 52800, 'f32', True, True),
    ('stats', 32, 10368, 'bf16', False, False),
    ('stats', 32, 10368, 'f16', False, False),
    ('stats', 32, 10368, 'f32', False, False),
    ('stats', 32, 110592, 'bf16', False, False),
    ('stats', 32, 110592, 'f16', False, False),
    ('stats', 32, 110592, 'f32', False, False),
    ('stats', 32, 116736, 'bf16', False, False),
    ('stats', 32, 116736, 'f16', False, False),
    ('stats', 32, 116736, 'f32', False, False),
    ('stats', 32, 12288, 'bf16', False, False),
    ('stats', 32, 12288, 'f16', False, False),
    ('stats', 32, 12288, 'f32', False, False),
    ('stats', 32, 12544, 'bf16', False, False),
    ('stats', 32, 12544, 'f16', False, False),
    ('stats', 32, 12544, 'f32', False, False),
    ('stats', 32, 1296, 'bf16', False, False),
    ('stats', 32, 1296, 'f16', False, False),
    ('stats', 32, 1296, 'f32', False, False),
    ('stats', 32, 13440, 'bf16', False, False),
    ('stats', 32, 13440, 'f16', False, False),
    ('stats', 32, 13440, 'f32', False, False),
    ('stats', 32, 13824, 'bf16', False, False),
    ('stats', 32, 13824, 'f16', False, False),
    ('stats', 32, 13824, 'f32', False, False),
    ('stats', 32, 14400, 'bf16', False, False),
    ('stats', 32, 14400, 'f16', False, False),
    ('stats', 32, 14400, 'f32', False, False),
    ('stats', 32, 14592, 'bf16', False, False),
    ('stats', 32, 14592, 'f16', False, False),
    ('stats', 32, 14592, 'f32', False, False),
    ('stats', 32, 1536, 'bf16', False, False),
    ('stats', 32, 1536, 'f16', False, False),
    ('stats', 32, 1536, 'f32', False, False),
    ('stats', 32, 156800, 'bf16', False, False),
    ('stats', 32, 156800, 'f16', False, False),
    ('stats', 32, 156800, 'f32', False, False),
    ('stats', 32, 161280, 'bf16', False, False),
    ('stats', 32, 161280, 'f16', False, False),
    ('stats', 32, 161280, 'f32', False, False),
    ('stats', 32, 16384, 'bf16', False, False),
    ('stats', 32, 16384, 'f16', False, False),
    ('stats', 32, 16384, 'f32', False, False),
    ('stats', 32, 175104, 'bf16', False, False),
    ('stats', 32, 175104, 'f16', False, False),
    ('stats', 32, 175104, 'f32', False, False),
    ('stats', 32, 18432, 'bf16', False, False),
    ('stats', 32, 18432, 'f16', False, False),
    ('stats', 32, 18432, 'f32', False, False),
    ('stats', 32, 184832, 'bf16', False, False),
    ('stats', 32, 184832, 'f16', False, False),
    ('stats', 32, 184832, 'f32', False, False),
    ('stats', 32, 19600, 'bf16', False, False),
    ('stats', 32, 19600, 'f16', False, False),
    ('stats', 32, 19600, 'f32', False, False),
    ('stats', 32, 20160, 'bf16', False, False),
    ('stats', 32, 20160, 'f16', False, False),
    ('stats', 32, 20160, 'f32', False, False),
    ('stats', 32, 20736, 'bf16', False, False),
    ('stats', 32, 20736, 'f16', False, False),
    ('stats', 32, 20736, 'f32', False, False),
    ('stats', 32, 21888, 'bf16', False, False),
    ('stats', 32, 21888, 'f16', False, False),
    ('stats', 32, 21888, 'f32', False, False),
    ('stats', 32, 221184, 'bf16', False, False),
    ('stats', 32, 221184, 'f16', False, False),
    ('stats', 32, 221184, 'f32', False, False),
    ('stats', 32, 2304, 'bf16', False, False),
    ('stats', 32, 2304, 'f16', False, False),
    ('stats', 32, 2304, 'f32', False, False),
    ('stats', 32, 23104, 'bf16', False, False),
    ('stats', 32, 23104, 'f16', False, False),
    ('stats', 32, 23104, 'f32', False, False),
    ('stats', 32, 233472, 'bf16', False, False),
    ('stats', 32, 233472, 'f16', False, False),
    ('stats', 32, 233472, 'f32', False, False),
    ('stats', 32, 24576, 'bf16', False, False),
    ('stats', 32, 24576, 'f16', False, False),
    ('stats', 32, 24576, 'f32', False, False),
    ('stats', 32, 25088, 'bf16', False, False),
    ('stats', 32, 25088, 'f16', False, False),
    ('stats', 32, 25088, 'f32', False, False),
    ('stats', 32, 2592, 'bf16', False, False),
    ('stats', 32, 2592, 'f16', False, False),
    ('stats', 32, 2592, 'f32', False, False),
    ('stats', 32, 26880, 'bf16', False, False),
    ('stats', 32, 26880, 'f16', False, False),
    ('stats', 32, 26880, 'f32', False, False),
    ('stats', 32, 28800, 'bf16', False, False),
    ('stats', 32, 28800, 'f16', False, False),
    ('stats', 32, 28800, 'f32', False, False),
    ('stats', 32, 3072, 'bf16', False, False),
    ('stats', 32, 3072, 'f16', False, False),
    ('stats', 32, 3072, 'f32', False, False),
    ('stats', 32, 3136, 'bf16', False, False),
    ('stats', 32, 3136, 'f16', False, False),
    ('stats', 32, 3136, 'f32', False, False),
    ('stats', 32, 313600, 'bf16', False, False),
    ('stats', 32, 313600, 'f16', False, False),
    ('stats', 32, 313600, 'f32', False, False),
    ('stats', 32, 322560, 'bf16', False, False),
    ('stats', 32, 322560, 'f16', False, False),
    ('stats', 32, 322560, 'f32', False, False),
    ('stats', 32, 32768, 'bf16', False, False),
    ('stats', 32, 32768, 'f16', False, False),
    ('stats', 32, 32768, 'f32', False, False),
    ('stats', 32, 3360, 'bf16', False, False),
    ('stats', 32, 3360, 'f16', False, False),
    ('stats', 32, 3360, 'f32', False, False),
    ('stats', 32, 350208, 'bf16', False, False),
    ('stats', 32, 350208, 'f16', False, False),
    ('stats', 32, 350208, 'f32', False, False),
    ('stats', 32, 3600, 'bf16', False, False),
    ('stats', 32, 3600, 'f16', False, False),
    ('stats', 32, 3600, 'f32', False, False),
    ('stats', 32, 36864, 'bf16', False, False),
    ('stats', 32, 36864, 'f16', False, False),
    ('stats', 32, 36864, 'f32', False, False),
    ('stats', 32, 369664, 'bf16', False, False),
    ('stats', 32, 369664, 'f16', False, False),
    ('stats', 32, 369664, 'f32', False, False),
    ('stats', 32, 4096, 'bf16', False, False),
    ('stats', 32, 4096, 'f16', False, False),
    ('stats', 32, 4096, 'f32', False, False),
    ('stats', 32, 442368, 'bf16', False, False),
    ('stats', 32, 442368, 'f16', False, False),
    ('stats', 32, 442368, 'f32', False, False),
    ('stats', 32, 4608, 'bf16', False, False),
    ('stats', 32, 4608, 'f16', False, False),
    ('stats', 32, 4608, 'f32', False, False),
    ('stats', 32, 466944, 'bf16', False, False),
    ('stats', 32, 466944, 'f16', False, False),
    ('stats', 32, 466944, 'f32', False, False),
    ('stats', 32, 49152, 'bf16', False, False),
    ('stats', 32, 49152, 'f16', False, False),
    ('stats', 32, 49152, 'f32', False, False),
    ('stats', 32, 50176, 'bf16', False, False),
    ('stats', 32, 50176, 'f16', False, False),
    ('stats', 32, 50176, 'f32', False, False),
    ('stats', 32, 5184, 'bf16', False, False),
    ('stats', 32, 5184, 'f16', False, False),
    ('stats', 32, 5184, 'f32', False, False),
    ('stats', 32, 53760, 'bf16', False, False),
    ('stats', 32, 53760, 'f16', False, False),
    ('stats', 32, 53760, 'f32', False, False),
    ('stats', 32, 55296, 'bf16', False, False),
    ('stats', 32, 55296, 'f16', False, False),
    ('stats', 32, 55296, 'f32', False, False),
    ('stats', 32, 57600, 'bf16', False, False),
    ('stats', 32, 57600, 'f16', False, False),
    ('stats', 32, 57600, 'f32', False, False),
    ('stats', 32, 58368, 'bf16', False, False),
    ('stats', 32, 58368, 'f16', False, False),
    ('stats', 32, 58368, 'f32', False, False),
    ('stats', 32, 6144, 'bf16', False, False),
    ('stats', 32, 6144, 'f16', False, False),
    ('stats', 32, 6144, 'f32', False, False),
    ('stats', 32, 6272, 'bf16', False, False),
    ('stats', 32, 6272, 'f16', False, False),
    ('stats', 32, 6272, 'f32', False, False),
    ('stats', 32, 627200, 'bf16', False, False),
    ('stats', 32, 627200, 'f16', False, False),
    ('stats', 32, 627200, 'f32', False, False),
    ('stats', 32, 645120, 'bf16', False, False),
    ('stats', 32, 645120, 'f16', False, False),
    ('stats', 32, 645120, 'f32', False, False),
    ('stats', 32, 65536, 'bf16', False, False),
    ('stats', 32, 65536, 'f16', False, False),
    ('stats', 32, 65536, 'f32', False, False),
    ('stats', 32, 6720, 'bf16', False, False),
    ('stats', 32, 6720, 'f16', False, False),
    ('stats', 32, 6720, 'f32', False, False),
    ('stats', 32, 700416, 'bf16', False, False),
    ('stats', 32, 700416, 'f16', False, False),
    ('stats', 32, 700416, 'f32', False, False),
    ('stats', 32, 7200, 'bf16', False, False),
    ('stats', 32, 7200, 'f16', False, False),
    ('stats', 32, 7200, 'f32', False, False),
    ('stats', 32, 739328, 'bf16', False, False),
    ('stats', 32, 739328, 'f16', False, False),
    ('stats', 32, 739328, 'f32', False, False),
    ('stats', 32, 768, 'bf16', False, False),
    ('stats', 32, 768, 'f16', False, False),
    ('stats', 32, 768, 'f32', False, False),
    ('stats', 32, 78400, 'bf16', False, False),
    ('stats', 32, 78400, 'f16', False, False),
    ('stats', 32, 78400, 'f32', False, False),
    ('stats', 32, 80640, 'bf16', False, False),
    ('stats', 32, 80640, 'f16', False, False),
    ('stats', 32, 80640, 'f32', False, False),
    ('stats', 32, 8192, 'bf16', False, False),
    ('stats', 32, 8192, 'f16', False, False),
    ('stats', 32, 8192, 'f32', False, False),
    ('stats', 32, 87552, 'bf16', False, False),
    ('stats', 32, 87552, 'f16', False, False),
    ('stats', 32, 87552, 'f32', False, False),
    ('stats', 32, 9216, 'bf16', False, False),
    ('stats', 32, 9216, 'f16', False, False),
    ('stats', 32, 9216, 'f32', False, False),
    ('stats', 32, 92416, 'bf16', False, False),
    ('stats', 32, 92416, 'f16', False, False),
    ('stats', 32, 92416, 'f32', False, False),
    ('stats', 32, 98304, 'bf16', False, False),
    ('stats', 32, 98304, 'f16', False, False),
    ('stats', 32, 98304, 'f32', False, False),
    ('stats', 4, 192, 'bf16', True, False),
    ('stats', 4, 192, 'f16', True, False),
    ('stats', 4, 192, 'f32', True, False),
    ('stats', 4, 2080, 'bf16', True, True),
    ('stats', 4, 2080, 'f16', True, True),
    ('stats', 4, 2080, 'f32', True, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_census_signatures_against_float64(dn):
    dt = DTS[dn]
    sigs = [s for s in CENSUS if s[3 if s[0] == "stats" else 4] == dn]
    assert sigs
    for i, s in enumerate(sigs):
        if s[0] == "stats":
            _, nseg, seg_len, _, unbiased, mm = s
            x = _randn((nseg * seg_len,), 700 + i, 1.3, 0.4).to(dt)
            _check_stats(x, nseg, seg_len, unbiased, f"census {s}", minmax=mm)
        else:
            _, B, C, HW, _, groups, per_batch, has_g, has_b, act = s
            ns = B * groups if per_batch else groups
            x = _randn((B, C, HW), 700 + i, 1.5, 0.2).to(dt)
            y = torch.empty_like(x)
            mean, var = _randn((ns,), 800 + i, 0.4), _randn((ns,), 900 + i, 0.5).abs() + 0.3
            gamma = _randn((C,), 1000 + i, 0.5, 1.0) if has_g else None
            beta = _randn((C,), 1100 + i, 0.3) if has_b else None
            assert _apply_call(x, y, B, C, HW, groups, mean, var, per_batch, gamma, beta, act) == OK, _err()
            ref, bound = _apply64(x, mean, var, gamma, beta, act, groups, per_batch)
            _within(y, ref, bound, "gn_apply", dt, f"census {s}")


@pytest.mark.gpu
def test_census_is_complete():
    got = record_census()
    missing = sorted(set(got) - set(CENSUS), key=repr)
    assert not missing, f"{len(missing)} signatures not in CENSUS: {missing}"


# ---------------------------------------------------------------------------------------------------------------------
# report
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_zz_report_worst_ratios():
    """Prints the worst err / bound per family and dtype seen by the tests above (run with -s)."""
    for (fam, dn), r in sorted(WORST.items()):
        print(f"worst err/bound {fam:10s} {dn:5s} {r:.3g}")
