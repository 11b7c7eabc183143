"""The tensor-core VAE kernels (csrc/td_conv.cu, csrc/td_attn.cu, csrc/td_nhwc.cu) per element against float64, in fp16
and bf16, at the layer shapes the autoencoder issues.

Every reference is computed in float64 on the GPU from the exact 16-bit inputs, together with the magnitude sum its
error bound needs.  Each output element must satisfy its own bound, so a wrong value where outputs are small fails as
surely as one at the largest output.

Bounds (u_out: unit roundoff of the output format, 2^-11 fp16 / 2^-8 bf16; tau: half the smallest subnormal spacing,
2^-25 fp16 / 2^-134 bf16; e32 = 2^-24, the fp32 unit roundoff):

  conv / GEMM    v = alpha * sum a w + bias (+ residual), the fp32 value before rounding:
                 |v_fp32 - v| <= gamma * |alpha| * S + 2 e32 (|alpha| S + |bias| + |residual|),   S = sum |a w|,
                 gamma = K * 2^-22 for K products.  gamma is an ASSUMPTION about the wgmma fp32 accumulation (it is
                 not IEEE round-to-nearest; the bound allows two fp32 ulps per term), not a measurement.  The two e32
                 terms are the epilogue's fmaf(acc, alpha, bias) and the residual add; the residual itself is an
                 exact 16-bit input.  Output: |got - ref| <= u_out |ref| + (1 + u_out) e + tau.
  post           t = v * scale + shift (one fmaf): e_t = |scale| e_v + e32 |t|.  With SiLU (|silu'| <= 1.0998):
                 e = 1.1 e_t + (eps_exp(t) sigma(-t) + e32 + 2^-22) |silu(t)| + [t < -87] 2^-119, where
                 eps_exp(t) = (2 + floor(1.173 |t|)) 2^-23 is __expf's documented error, 2^-22 is __fdividef's two
                 ulps, and the last term is __fdividef's documented result 0 for divisors above 2^126 (t < -87.3,
                 where |silu(t)| < 2^-119).
  up2            the reference is the four parity 2x2 convolutions over the folded 16-bit taps themselves
                 (fold_upsample_weight), so the plain conv bound applies with K = 4 Cin.
  attention      see `_attention64`.
  softmax_rows   see `_softmax64`.
  gn_apply       see `_gn_apply64`; gn_stats uses the tolerances of the existing statistics tests.
  layout, upsample, wrap: bit-exact.
"""
import contextlib
import ctypes
import copy
import inspect
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_blend_limits import launched, template_args

DTS = {"f16": torch.float16, "bf16": torch.bfloat16}
DN = list(DTS)
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
TAU = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134}
E32 = 2.0 ** -24
G_ACC = 2.0 ** -22
WORST = {}          # (family, dtype name) -> worst err / bound seen


def _ops():
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops
    return vae_ops


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def _randn(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * scale + shift


def _pitched(t, extra, fill=float("nan")):
    """t [..., C] inside a buffer `extra` columns wider, the padding filled with `fill` (NaN: must never be read)."""
    if extra == 0:
        return t.contiguous()
    buf = torch.full((*t.shape[:-1], t.shape[-1] + extra), fill, dtype=t.dtype, device=t.device)
    buf[..., :t.shape[-1]] = t
    return buf[..., :t.shape[-1]]


def _name(dt):
    return "f16" if dt == torch.float16 else "bf16"


def _note(family, dt, ratio):
    key = (family, _name(dt))
    WORST[key] = max(WORST.get(key, 0.0), ratio)


def _out_bound(ref, e, dt):
    return U[dt] * ref.abs() + (1.0 + U[dt]) * e + TAU[dt]


def _violations(got, ref, bound):
    return int(((got.double() - ref).abs() > bound).sum())


def _within(got, ref, bound, family, dt, what):
    g = got.double()
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    ratio = (g - ref).abs() / bound
    worst = ratio.max().item()
    _note(family, dt, worst)
    if worst > 1.0:
        i = int(ratio.argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        raise AssertionError(f"{what}: {_violations(got, ref, bound)} elements over the bound; worst at {idx}: got {g[idx].item()!r} "
                             f"ref {ref[idx].item()!r} bound {bound[idx].item():.3g} (err / bound {worst:.3g})")
    return worst


# ------------------------------------------------------------------------------------------------ float64 references
def _conv64(x, w, k, stride, pad, oh, ow, cout):
    """x [N, H, W, Cin] (any pitch), w [k*k, >= cout, >= Cin] -> (sum a w, sum |a w|) float64 [N, oh, ow, cout]."""
    N, H, W, Cin = x.shape
    hb = max(0, stride * (oh - 1) + k - pad[0] - H)
    wb = max(0, stride * (ow - 1) + k - pad[1] - W)
    xp = F.pad(x.double(), (0, 0, pad[1], wb, pad[0], hb))
    ref = torch.zeros((N, oh, ow, cout), dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(ref)
    for ky in range(k):
        for kx in range(k):
            sl = xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride, :]
            wt = w[ky * k + kx, :cout, :Cin].double().t()
            ref += sl @ wt
            mag += sl.abs() @ wt.abs()
    return ref, mag


def _upconv64(x, w16, cout, swap_parity=False):
    """Nearest-2x upsample + 3x3 conv as the four parity 2x2 convolutions over the folded taps w16 [16, >= cout, Cin]."""
    N, H, W, Cin = x.shape
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    ref = torch.zeros((N, 2 * H, 2 * W, cout), dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(ref)
    for py in range(2):
        for px in range(2):
            acc = torch.zeros((N, H, W, cout), dtype=torch.float64, device=x.device)
            am = torch.zeros_like(acc)
            for ty in range(2):
                for tx in range(2):
                    sl = xp[:, py + ty:py + ty + H, px + tx:px + tx + W, :]
                    wt = w16[(py * 2 + px) * 4 + ty * 2 + tx, :cout, :Cin].double().t()
                    acc += sl @ wt
                    am += sl.abs() @ wt.abs()
            qx = 1 - px if swap_parity else px
            ref[:, py::2, qx::2] = acc
            mag[:, py::2, qx::2] = am
    return ref, mag


def _pre(ref, mag, K, alpha=1.0, bias=None, res=None):
    """(v, e_v): the float64 value before the output rounding and the bound on the kernel's fp32 error in it."""
    v = alpha * ref
    s = abs(alpha) * mag
    if bias is not None:
        v = v + bias
        s = s + bias.abs()
    if res is not None:
        v = v + res.double()
        s = s + res.double().abs()
    return v, K * G_ACC * abs(alpha) * mag + 2 * E32 * s


def _silu_err(t, z):
    eexp = (2.0 + torch.floor(1.173 * t.abs())) * 2.0 ** -23
    return (eexp * torch.sigmoid(-t) + E32 + 2.0 ** -22) * z.abs() + torch.where(t < -87.0, 2.0 ** -119, 0.0)


def _post64(v, e_v, scale, shift, act):
    s, h = scale.double(), shift.double()
    t = v * s + h
    e_t = s.abs() * e_v + E32 * t.abs()
    if not act:
        return t, e_t
    z = t * torch.sigmoid(t)
    return z, 1.1 * e_t + _silu_err(t, z)


# ------------------------------------------------------------------------------------------------ conv / GEMM cases
def _conv_case(dt, N, H, W, Cin, Cout, k, stride=1, seed=0, residual=False, post=None, dual=False, x_extra=0, w_extra=0, y_extra=0,
               r_extra=0, shift=None, w_rows=None, call=True):
    """One td_conv2d_nhwc call on random data; returns (got, want, bound[, got2, want2, bound2]) in NHWC.
    stride 2 is the ldm Downsample (no conv padding, output (H - 1) // 2 + 1)."""
    ops = _ops()
    if stride == 1:
        pad, oh, ow = (k // 2, k // 2), H, W
    else:
        pad, oh, ow = (0, 0), (H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1
    x = _pitched(_randn((N, H, W, Cin), seed, 0.7).to(dt), x_extra)
    w = _pitched(_randn((k * k, Cout, Cin), seed + 1, (Cin * k * k) ** -0.5).to(dt), w_extra)
    bias = _randn((Cout,), seed + 2, 0.3)
    res = _pitched(_randn((N, oh, ow, Cout), seed + 3, 0.5).to(dt), r_extra) if residual else None
    pst = None
    if post is not None:
        sh = _randn((Cout,), seed + 5, 0.2) if shift is None else shift
        pst = (_randn((Cout,), seed + 4, 0.4, 1.0), sh.contiguous(), bool(post))
    out = None
    if y_extra:
        out = _pitched(torch.empty((N, oh, ow, Cout), dtype=dt, device="cuda"), y_extra)
    got = ops.conv2d_nhwc(x, w, bias, ksize=k, stride=stride, pad=pad, out_hw=(oh, ow), residual=res, out=out, post=pst, dual=dual)
    ref, mag = _conv64(x, w, k, stride, pad, oh, ow, Cout)
    v, e = _pre(ref, mag, k * k * Cin, 1.0, bias.double(), res)
    raw = (v, _out_bound(v, e, dt))
    if pst is None:
        return got, raw[0], raw[1]
    z, ez = _post64(v, e, pst[0], pst[1], pst[2])
    if dual:
        return got[0], raw[0], raw[1], got[1], z, _out_bound(z, ez, dt)
    return got, z, _out_bound(z, ez, dt)


def _upconv_case(dt, N, H, W, Cin, Cout, seed=0, post=None, dual=False):
    ops = _ops()
    x = _randn((N, H, W, Cin), seed, 0.7).to(dt)
    w16 = ops.fold_upsample_weight(_randn((Cout, Cin, 3, 3), seed + 1, (Cin * 9) ** -0.5).to(dt), dt, cin_pad=Cin)
    bias = _randn((Cout,), seed + 2, 0.3)
    pst = (_randn((Cout,), seed + 4, 0.4, 1.0), _randn((Cout,), seed + 5, 0.2), bool(post)) if post is not None else None
    got = ops.upconv2x_nhwc(x, w16, bias, post=pst, dual=dual)
    ref, mag = _upconv64(x, w16, Cout)
    v, e = _pre(ref, mag, 4 * Cin, 1.0, bias.double())
    if pst is None:
        return got, v, _out_bound(v, e, dt), (x, w16, bias)
    z, ez = _post64(v, e, pst[0], pst[1], pst[2])
    if dual:
        return got, (v, _out_bound(v, e, dt)), (z, _out_bound(z, ez, dt)), (x, w16, bias, pst)
    return got, z, _out_bound(z, ez, dt), (x, w16, bias)


def _gemm_case(dt, M, K, n, seed=0, a_pitch=None, b_rows=None, b_pitch=None, y_pitch=None, alpha=1.0, bias=True, bias_per_row=False,
               guard=0):
    """vae_ops.gemm_nt with NaN in every padding column of A / B / D and in `guard` rows past M; returns
    (got, want, bound, out buffer, M)."""
    ops = _ops()
    a = _pitched(_randn((M, K), seed, 0.5).to(dt), (a_pitch or K) - K)
    b = _pitched(_randn((b_rows or n, K), seed + 1, K ** -0.5).to(dt), (b_pitch or K) - K)
    bv = _randn((M if bias_per_row else n,), seed + 2, 0.3) if bias else None
    yp = y_pitch or ops.round_up(n, 8)
    obuf = torch.full((M + guard, yp), float("nan"), dtype=dt, device="cuda")
    got = ops.gemm_nt(a, b, bias=bv, alpha=alpha, n=n, out=obuf[:M, :n], bias_per_row=bias_per_row)
    ref = a.double() @ b[:n].double().t()
    mag = a.double().abs() @ b[:n].double().abs().t()
    bb = None if bv is None else (bv.double()[:, None] if bias_per_row else bv.double()[None, :])
    v, e = _pre(ref, mag, K, alpha, bb)
    return got, v, _out_bound(v, e, dt), obuf, M


def _assert_nan_kept(buf, region, what):
    """Every element of `buf` outside `region` (a boolean mask of what the kernel may write) is still NaN."""
    outside = buf[~region]
    assert torch.isnan(outside.float()).all(), f"{what}: the kernel wrote {int((~torch.isnan(outside.float())).sum())} padding / guard elements"


# ------------------------------------------------------------------------------------------------ attention / softmax / GN
def _attention64(q, k, v, alpha, dt, rows=256, stale_max=False, qidx=None):
    """Float64 softmax(alpha q k^T) v and its per-element bound, `rows` queries at a time (no T x T matrix for large T);
    qidx: only these query rows (the output has one row per index), against all T keys.

    The kernel computes S in fp32 (products over C: gamma_C = C 2^-22 per |q||k| sum; the two warpgroup partials'
    add, the scale by alpha log2(e) and that constant: 4 e32 |S| more), so the logit of key j is off by at most
    D_j = alpha (gamma_C sum_c |q_c k_jc| + 4 e32 |S_j|) (natural-log units).  p_j = exp2(logit_j - max) is then
    relatively off by E = expm1(2 max_j D_j + e32 max_j |L_j - L_max| + 2^-22) (the row max carries one D, the
    subtraction one e32, exp2f two ulps).  Before P V, p_j is rounded to 16 bits (u_in; plus an absolute 2^-25 where
    fp16 p falls into subnormals, relative to the running max, which the final normalisation only shrinks).  Each of
    the ceil(T / 64) key blocks rescales the accumulators by exp2f(m_old - m_new) (2 ulps) and one multiply (e32).
    P V and the row sum accumulate T terms in fp32 (T 2^-22, T e32).  The row sum uses the unrounded p, so its
    relative error is at most E plus its accumulation; numerator and denominator together give
        kappa = u_in + 2 E + 2 blocks (2^-22 + e32) + T 2^-22 + T e32 + 2^-22 (the final 1 / l and product),
        |got - ref| <= u_out |ref| + (1 + u_out) (kappa sum_j p_j |v_j| + tau_P sum_j |v_j| / l) + tau.
    stale_max: the mutated reference of an online softmax that never rescales earlier key blocks."""
    T, C = k.shape
    alpha = float(torch.tensor(alpha, dtype=torch.float32))
    qd, kd, vd = (q if qidx is None else q[qidx]).double(), k.double(), v.double()
    kabs, vabs = kd.abs(), vd.abs()
    vsum = vabs.sum(0, keepdim=True)
    out = torch.empty((qd.shape[0], C), dtype=torch.float64, device=q.device)
    bnd = torch.empty_like(out)
    blocks = (T + 63) // 64
    tau_p = 2.0 ** -25 if dt == torch.float16 else 0.0
    for r0 in range(0, qd.shape[0], rows):
        S = qd[r0:r0 + rows] @ kd.t()
        Sabs = qd[r0:r0 + rows].abs() @ kabs.t()
        L = alpha * S
        m = L.max(1, keepdim=True).values
        e = torch.exp(L - m)
        l = e.sum(1, keepdim=True)
        p = e / l
        if stale_max:
            num = torch.zeros((S.shape[0], C), dtype=torch.float64, device=q.device)
            den = torch.zeros((S.shape[0], 1), dtype=torch.float64, device=q.device)
            for b0 in range(0, T, 64):
                Lb = L[:, b0:b0 + 64]
                eb = torch.exp(Lb - Lb.max(1, keepdim=True).values)
                num += eb @ vd[b0:b0 + 64]
                den += eb.sum(1, keepdim=True)
            ref = num / den
        else:
            ref = p @ vd
        pv = p @ vabs
        D = alpha * (C * G_ACC * Sabs + 4 * E32 * S.abs())
        E = torch.expm1(2 * D.max(1, keepdim=True).values + E32 * (L - m).abs().max(1, keepdim=True).values + 2.0 ** -22)
        kappa = U[dt] + 2 * E + 2 * blocks * (2.0 ** -22 + E32) + T * G_ACC + T * E32 + 2.0 ** -22
        out[r0:r0 + rows] = ref
        bnd[r0:r0 + rows] = _out_bound(ref, kappa * pv + tau_p * vsum / l, dt)
    return out, bnd


def _qkv(T, C, dt, seed):
    """q, k of std 1.7 (logits alpha q.k of std ~2.9: a softmax far from uniform), v of std 1."""
    return (_randn((T, C), seed, 1.7).to(dt), _randn((T, C), seed + 1, 1.7, 0.2).to(dt), _randn((T, C), seed + 2).to(dt))


def _softmax64(x, cols, dt):
    """Float64 row softmax of x[:, :cols] and its bound.  The kernel: __expf(x - m) ((2 + floor(1.173 |x - m|)) ulps),
    a running fp32 sum (cols + 64 additions incl. the merges: (cols + 64) e32) whose per-thread, warp and CTA merges
    rescale by __expf of a max difference (at most ceil(pitch / 2048) + 13 merges of (2 + floor(1.173 R)) ulps, R the
    row's range), 1 / sum and the product (3 ulps)."""
    xd = x[:, :cols].double()
    m = xd.max(1, keepdim=True).values
    R = (m - xd.min(1, keepdim=True).values)
    e = torch.exp(xd - m)
    ref = e / e.sum(1, keepdim=True)
    merges = math.ceil(x.shape[1] / 2048) + 13
    eps_sum = (cols + 64) * E32 + merges * (2.0 + torch.floor(1.173 * R)) * 2.0 ** -23
    eexp = (2.0 + torch.floor(1.173 * (xd - m).abs())) * 2.0 ** -23
    return ref, _out_bound(ref, ref * (eexp + eps_sum + 3 * 2.0 ** -23), dt)


def _gn_apply64(x, mean, var, gamma, beta, act, dt, eps=1e-6, groups=32):
    """y = act((x - mean) rstd gamma + beta) from the given fp32 statistics.  The kernel folds it into sc = rstd gamma
    (var + eps, sqrtf, 1 / s, * gamma: 5 ulps) and sh = fmaf(-mean, sc, beta), then fmaf(x, sc, sh):
    e_t = 5 2^-23 (|x| + |mean|) |sc| + e32 (|sh| + |t|), then SiLU as in the conv epilogue."""
    C = x.shape[-1]
    cpg = C // groups
    md = mean.double().repeat_interleave(cpg)
    rstd = 1.0 / torch.sqrt(var.double().repeat_interleave(cpg) + float(torch.tensor(eps, dtype=torch.float32)))
    sc = rstd * (gamma.double() if gamma is not None else 1.0)
    sh = -md * sc + (beta.double() if beta is not None else 0.0)
    xd = x.double()
    t = xd * sc + sh
    e_t = 5 * 2.0 ** -23 * (xd.abs() + md.abs()) * sc.abs() + E32 * (sh.abs() + t.abs())
    if not act:
        return t, _out_bound(t, e_t, dt)
    z = t * torch.sigmoid(t)
    return z, _out_bound(z, 1.1 * e_t + _silu_err(t, z), dt)


# ------------------------------------------------------------------------------------------------ 1. which form ran
def _bn(cout):
    bn = 256
    if cout < 256:
        bn = 16
        while bn < cout:
            bn *= 2
    return bn


# (name, tile the kernel picks, builder) -- one per pixel-tile shape; together they reach every BN
FORM_CASES = [
    ("16x8", 3, lambda dt: _conv_case(dt, 1, 20, 36, 64, 3, 3, seed=11, y_extra=5)),
    ("8x16_s1", 17, lambda dt: _conv_case(dt, 1, 21, 9, 64, 17, 3, seed=12, y_extra=7)),
    ("8x16_s2", 64, lambda dt: _conv_case(dt, 1, 29, 23, 128, 64, 3, stride=2, seed=13, residual=True)),
    ("128x1", 128, lambda dt: _gemm_case(dt, 300, 200, 128, seed=14, a_pitch=256, b_pitch=256)[:3]),
    ("up2", 512, lambda dt: _upconv_case(dt, 1, 13, 21, 64, 512, seed=15)[:3]),
]


@pytest.mark.gpu
def test_every_conv_form_is_reached_and_correct():
    """Each case must launch exactly the conv_gemm_kernel<BN, BF16> instantiation its Cout selects and meet the bound;
    together the cases must reach all 10 instantiations and every pixel-tile shape in both dtypes."""
    reached, tiles = set(), set()
    for dn, dt in DTS.items():
        for name, cout, build in FORM_CASES:
            box = {}

            def run():
                box["r"] = build(dt)
            names = launched(run)
            forms = {tuple(f) for f in template_args(names, "conv_gemm_kernel")}
            want = (str(_bn(cout)), "true" if dt == torch.bfloat16 else "false")
            assert forms == {want}, f"{name} {dn}: launched {sorted(forms)}, expected {want}"
            got, ref, bound = box["r"]
            _within(got, ref, bound, "conv", dt, f"form {name} {dn}")
            reached.add((_bn(cout), dt))
            tiles.add((name, dt))
    assert reached == {(bn, dt) for bn in (16, 32, 64, 128, 256) for dt in DTS.values()}, sorted(map(str, reached))
    assert tiles == {(n, dt) for n, *_ in FORM_CASES for dt in DTS.values()}


# ------------------------------------------------------------------------------------------------ 3. layer census
SPIED = ("conv2d_nhwc", "upconv2x_nhwc", "gemm_nt", "attention", "softmax_rows", "gn_stats_nhwc", "gn_apply_nhwc", "upsample2x_nhwc")


def _signature(name, fn, args, kw):
    ops = _ops()
    A = inspect.signature(fn).bind(*args, **kw)
    A.apply_defaults()
    a = A.arguments
    if name == "conv2d_nhwc":
        x, w = a["x"], a["w"]
        N, H, W, Cin = x.shape
        oh, ow = a["out_hw"] if a["out_hw"] is not None else (H, W)
        cout = a["cout"] or w.shape[1]
        res, post = a["residual"], a["post"]
        return ("conv", N, H, W, Cin, x.stride(2), cout, w.shape[1], a["ksize"], a["stride"], a["pad"][0], a["pad"][1], oh, ow,
                res.stride(2) if res is not None else 0, -1 if post is None else int(bool(post[2])), bool(a["dual"]),
                a["out"].stride(2) if a["out"] is not None else cout, bool(a["bias_per_row"]))
    if name == "upconv2x_nhwc":
        x, w16, post = a["x"], a["w16"], a["post"]
        return ("up2", *x.shape, a["cout"] or w16.shape[1], -1 if post is None else int(bool(post[2])), bool(a["dual"]))
    if name == "gemm_nt":
        A_, B_ = a["a"], a["b"]
        nb = a["n"] or B_.shape[0]
        return ("gemm", A_.shape[0], A_.shape[1], A_.stride(0), nb, B_.shape[0], B_.stride(0),
                a["out"].stride(0) if a["out"] is not None else ops.round_up(nb, 8), float(a["alpha"]), a["bias"] is not None,
                bool(a["bias_per_row"]))
    if name == "attention":
        q = a["q"]
        return ("attn", q.shape[0], q.shape[1], q.stride(0), a["k"].stride(0), a["v"].stride(0), float(a["alpha"]))
    if name == "softmax_rows":
        x = a["x"]
        return ("softmax", x.shape[0], x.shape[1], a["cols"], a["out"] is x)
    if name == "gn_stats_nhwc":
        x = a["x"]
        return ("gn_stats", x.shape[1], x.shape[2], x.shape[3], a["groups"])
    if name == "gn_apply_nhwc":
        x = a["x"]
        return ("gn_apply", x.shape[1], x.shape[2], x.shape[3], a["gamma"] is not None, a["beta"] is not None, bool(a["act"]))
    x = a["x"]
    return ("up_nn", *x.shape)


def _sd_width_net(is_dec, seed):
    """Full-width SD autoencoder half (ch=128, ch_mult (1,2,4,4), 2 res blocks), as in test_gpu_vae.py."""
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), seed)
    net.eval()
    net.original_forward = net.forward
    return net


# decoder 40 x 52 latent at tile 16 and encoder 200 x 264 image at tile 64: the encoder's deepest level has tiles
# narrower than 16 pixels (the 8 x 16 pixel tile), both have wider ones
CENSUS_RUNS = [(True, 40, 52, 16), (False, 200, 264, 64)]


@contextlib.contextmanager
def census_spy():
    """While active, the signature of every vae_engine.ops call in SPIED is added to the yielded set."""
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    seen = set()
    real = {n: getattr(ve.ops, n) for n in SPIED}

    def spy(n):
        def f(*a, **kw):
            seen.add(_signature(n, real[n], a, kw))
            return real[n](*a, **kw)
        return f
    try:
        for n in SPIED:
            setattr(ve.ops, n, spy(n))
        yield seen
    finally:
        for n in SPIED:
            setattr(ve.ops, n, real[n])


def record_census(runs=CENSUS_RUNS, dtypes=tuple(DTS.values())):
    """Distinct call signatures TensorCoreBackend issues for the SD-width encoder and decoder, fp16 and bf16, fast and
    slow mode.  runs: (is_decoder, H, W, tile[, one_tile]); one_tile: the input is exactly one padded tile, run through
    vae_tile_forward (VAEHook.__call__ runs an input that small through the network untiled)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from oracle import synth
    with census_spy() as seen:
        for is_dec, H, W, tile, *one in runs:
            base = _sd_width_net(is_dec, 3 if is_dec else 4)
            for dt in dtypes:
                net = copy.deepcopy(base).cuda().to(dt)
                z = synth.latent(5 if is_dec else 6, (1, 4 if is_dec else 3, H, W), dt).cuda()
                for fast in (True, False):
                    hook = tilevae.VAEHook(net, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
                    with torch.no_grad():
                        out = hook.vae_tile_forward(z) if one and one[0] else hook(z)
                    assert hook.backend_name == "wgmma"
                    del out
                del net, z
                torch.cuda.empty_cache()
    return sorted(seen, key=repr)


# recorded by record_census() on an H100 (fp16 and bf16, fast and slow mode, CENSUS_RUNS)
CENSUS = [
    ('conv', 1, 12, 16, 256, 256, 512, 512, 1, 1, 0, 0, 12, 16, 0, -1, False, 512, False),
    ('conv', 1, 12, 16, 256, 256, 512, 512, 3, 1, 1, 1, 12, 16, 0, -1, False, 512, False),
    ('conv', 1, 12, 16, 512, 512, 512, 512, 1, 1, 0, 0, 12, 16, 512, -1, False, 512, False),
    ('conv', 1, 12, 16, 512, 512, 512, 512, 3, 1, 1, 1, 12, 16, 0, -1, False, 512, False),
    ('conv', 1, 12, 16, 512, 512, 512, 512, 3, 1, 1, 1, 12, 16, 512, -1, False, 512, False),
    ('conv', 1, 12, 16, 512, 512, 512, 512, 3, 2, 0, 0, 6, 8, 0, -1, False, 512, False),
    ('conv', 1, 12, 16, 64, 64, 512, 512, 3, 1, 1, 1, 12, 16, 0, -1, False, 512, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 1, 1, 1, 128, 128, 0, -1, False, 128, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 1, 1, 1, 128, 128, 0, 1, False, 128, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 1, 1, 1, 128, 128, 128, -1, False, 128, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 1, 1, 1, 128, 128, 128, 1, True, 128, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 2, 0, 0, 64, 64, 0, -1, False, 128, False),
    ('conv', 1, 128, 128, 128, 128, 128, 128, 3, 2, 0, 0, 64, 64, 0, 1, True, 128, False),
    ('conv', 1, 128, 128, 64, 64, 128, 128, 3, 1, 1, 1, 128, 128, 0, -1, False, 128, False),
    ('conv', 1, 128, 128, 64, 64, 128, 128, 3, 1, 1, 1, 128, 128, 0, 1, True, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 1, 1, 1, 128, 72, 0, -1, False, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 1, 1, 1, 128, 72, 0, 1, False, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 1, 1, 1, 128, 72, 128, -1, False, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 1, 1, 1, 128, 72, 128, 1, True, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 2, 0, 0, 64, 36, 0, -1, False, 128, False),
    ('conv', 1, 128, 72, 128, 128, 128, 128, 3, 2, 0, 0, 64, 36, 0, 1, True, 128, False),
    ('conv', 1, 128, 72, 64, 64, 128, 128, 3, 1, 1, 1, 128, 72, 0, -1, False, 128, False),
    ('conv', 1, 128, 72, 64, 64, 128, 128, 3, 1, 1, 1, 128, 72, 0, 1, True, 128, False),
    ('conv', 1, 152, 144, 256, 256, 256, 256, 3, 1, 1, 1, 152, 144, 0, -1, False, 256, False),
    ('conv', 1, 152, 144, 256, 256, 256, 256, 3, 1, 1, 1, 152, 144, 0, 1, False, 256, False),
    ('conv', 1, 152, 144, 256, 256, 256, 256, 3, 1, 1, 1, 152, 144, 256, -1, False, 256, False),
    ('conv', 1, 152, 144, 256, 256, 256, 256, 3, 1, 1, 1, 152, 144, 256, 1, True, 256, False),
    ('conv', 1, 152, 144, 512, 512, 256, 256, 1, 1, 0, 0, 152, 144, 0, -1, False, 256, False),
    ('conv', 1, 152, 144, 512, 512, 256, 256, 3, 1, 1, 1, 152, 144, 0, -1, False, 256, False),
    ('conv', 1, 152, 144, 512, 512, 256, 256, 3, 1, 1, 1, 152, 144, 0, 1, False, 256, False),
    ('conv', 1, 152, 152, 256, 256, 256, 256, 3, 1, 1, 1, 152, 152, 0, -1, False, 256, False),
    ('conv', 1, 152, 152, 256, 256, 256, 256, 3, 1, 1, 1, 152, 152, 0, 1, False, 256, False),
    ('conv', 1, 152, 152, 256, 256, 256, 256, 3, 1, 1, 1, 152, 152, 256, -1, False, 256, False),
    ('conv', 1, 152, 152, 256, 256, 256, 256, 3, 1, 1, 1, 152, 152, 256, 1, True, 256, False),
    ('conv', 1, 152, 152, 512, 512, 256, 256, 1, 1, 0, 0, 152, 152, 0, -1, False, 256, False),
    ('conv', 1, 152, 152, 512, 512, 256, 256, 3, 1, 1, 1, 152, 152, 0, -1, False, 256, False),
    ('conv', 1, 152, 152, 512, 512, 256, 256, 3, 1, 1, 1, 152, 152, 0, 1, False, 256, False),
    ('conv', 1, 16, 16, 512, 512, 16, 16, 3, 1, 1, 1, 16, 16, 0, -1, False, 16, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 1, 1, 0, 0, 16, 16, 512, -1, False, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 1, 1, 0, 0, 16, 16, 512, 1, True, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 0, -1, False, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 0, 1, False, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 512, -1, False, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 512, 0, True, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 512, 1, False, 512, False),
    ('conv', 1, 16, 16, 512, 512, 512, 512, 3, 1, 1, 1, 16, 16, 512, 1, True, 512, False),
    ('conv', 1, 16, 9, 512, 512, 16, 16, 3, 1, 1, 1, 16, 9, 0, -1, False, 16, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 1, 1, 0, 0, 16, 9, 512, -1, False, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 1, 1, 0, 0, 16, 9, 512, 1, True, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 0, -1, False, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 0, 1, False, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 512, -1, False, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 512, 0, True, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 512, 1, False, 512, False),
    ('conv', 1, 16, 9, 512, 512, 512, 512, 3, 1, 1, 1, 16, 9, 512, 1, True, 512, False),
    ('conv', 1, 18, 18, 256, 256, 512, 512, 1, 1, 0, 0, 18, 18, 0, -1, False, 512, False),
    ('conv', 1, 18, 18, 256, 256, 512, 512, 3, 1, 1, 1, 18, 18, 0, -1, False, 512, False),
    ('conv', 1, 18, 18, 256, 256, 512, 512, 3, 1, 1, 1, 18, 18, 0, 1, False, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 1, 1, 1, 18, 18, 0, -1, False, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 1, 1, 1, 18, 18, 0, 1, False, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 1, 1, 1, 18, 18, 512, -1, False, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 1, 1, 1, 18, 18, 512, 1, True, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 2, 0, 0, 9, 9, 0, -1, False, 512, False),
    ('conv', 1, 18, 18, 512, 512, 512, 512, 3, 2, 0, 0, 9, 9, 0, 1, True, 512, False),
    ('conv', 1, 18, 32, 256, 256, 512, 512, 1, 1, 0, 0, 18, 32, 0, -1, False, 512, False),
    ('conv', 1, 18, 32, 256, 256, 512, 512, 3, 1, 1, 1, 18, 32, 0, -1, False, 512, False),
    ('conv', 1, 18, 32, 256, 256, 512, 512, 3, 1, 1, 1, 18, 32, 0, 1, False, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 1, 1, 1, 18, 32, 0, -1, False, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 1, 1, 1, 18, 32, 0, 1, False, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 1, 1, 1, 18, 32, 512, -1, False, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 1, 1, 1, 18, 32, 512, 1, True, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 2, 0, 0, 9, 16, 0, -1, False, 512, False),
    ('conv', 1, 18, 32, 512, 512, 512, 512, 3, 2, 0, 0, 9, 16, 0, 1, True, 512, False),
    ('conv', 1, 192, 288, 128, 128, 128, 128, 3, 1, 1, 1, 192, 288, 0, -1, False, 128, False),
    ('conv', 1, 192, 288, 128, 128, 128, 128, 3, 1, 1, 1, 192, 288, 0, 1, False, 128, False),
    ('conv', 1, 192, 288, 128, 128, 128, 128, 3, 1, 1, 1, 192, 288, 128, -1, False, 128, False),
    ('conv', 1, 192, 288, 128, 128, 128, 128, 3, 1, 1, 1, 192, 288, 128, 1, False, 128, False),
    ('conv', 1, 192, 288, 128, 128, 128, 128, 3, 1, 1, 1, 192, 288, 128, 1, True, 128, False),
    ('conv', 1, 192, 288, 128, 128, 16, 16, 3, 1, 1, 1, 192, 288, 0, -1, False, 16, False),
    ('conv', 1, 192, 288, 256, 256, 128, 128, 1, 1, 0, 0, 192, 288, 0, -1, False, 128, False),
    ('conv', 1, 192, 288, 256, 256, 128, 128, 3, 1, 1, 1, 192, 288, 0, -1, False, 128, False),
    ('conv', 1, 192, 288, 256, 256, 128, 128, 3, 1, 1, 1, 192, 288, 0, 1, False, 128, False),
    ('conv', 1, 192, 304, 128, 128, 128, 128, 3, 1, 1, 1, 192, 304, 0, -1, False, 128, False),
    ('conv', 1, 192, 304, 128, 128, 128, 128, 3, 1, 1, 1, 192, 304, 0, 1, False, 128, False),
    ('conv', 1, 192, 304, 128, 128, 128, 128, 3, 1, 1, 1, 192, 304, 128, -1, False, 128, False),
    ('conv', 1, 192, 304, 128, 128, 128, 128, 3, 1, 1, 1, 192, 304, 128, 1, False, 128, False),
    ('conv', 1, 192, 304, 128, 128, 128, 128, 3, 1, 1, 1, 192, 304, 128, 1, True, 128, False),
    ('conv', 1, 192, 304, 128, 128, 16, 16, 3, 1, 1, 1, 192, 304, 0, -1, False, 16, False),
    ('conv', 1, 192, 304, 256, 256, 128, 128, 1, 1, 0, 0, 192, 304, 0, -1, False, 128, False),
    ('conv', 1, 192, 304, 256, 256, 128, 128, 3, 1, 1, 1, 192, 304, 0, -1, False, 128, False),
    ('conv', 1, 192, 304, 256, 256, 128, 128, 3, 1, 1, 1, 192, 304, 0, 1, False, 128, False),
    ('conv', 1, 24, 32, 128, 128, 256, 256, 1, 1, 0, 0, 24, 32, 0, -1, False, 256, False),
    ('conv', 1, 24, 32, 128, 128, 256, 256, 3, 1, 1, 1, 24, 32, 0, -1, False, 256, False),
    ('conv', 1, 24, 32, 256, 256, 256, 256, 3, 1, 1, 1, 24, 32, 0, -1, False, 256, False),
    ('conv', 1, 24, 32, 256, 256, 256, 256, 3, 1, 1, 1, 24, 32, 256, -1, False, 256, False),
    ('conv', 1, 24, 32, 256, 256, 256, 256, 3, 2, 0, 0, 12, 16, 0, -1, False, 256, False),
    ('conv', 1, 24, 32, 512, 512, 512, 512, 3, 1, 1, 1, 24, 32, 0, -1, False, 512, False),
    ('conv', 1, 24, 32, 512, 512, 512, 512, 3, 1, 1, 1, 24, 32, 512, -1, False, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 1, 1, 0, 0, 24, 36, 512, -1, False, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 1, 1, 0, 0, 24, 36, 512, 1, True, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 3, 1, 1, 1, 24, 36, 0, -1, False, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 3, 1, 1, 1, 24, 36, 0, 1, False, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 3, 1, 1, 1, 24, 36, 512, -1, False, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 3, 1, 1, 1, 24, 36, 512, 0, True, 512, False),
    ('conv', 1, 24, 36, 512, 512, 512, 512, 3, 1, 1, 1, 24, 36, 512, 1, True, 512, False),
    ('conv', 1, 24, 36, 64, 64, 512, 512, 3, 1, 1, 1, 24, 36, 0, -1, False, 512, False),
    ('conv', 1, 24, 36, 64, 64, 512, 512, 3, 1, 1, 1, 24, 36, 0, 1, True, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 1, 1, 0, 0, 24, 38, 512, -1, False, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 1, 1, 0, 0, 24, 38, 512, 1, True, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 3, 1, 1, 1, 24, 38, 0, -1, False, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 3, 1, 1, 1, 24, 38, 0, 1, False, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 3, 1, 1, 1, 24, 38, 512, -1, False, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 3, 1, 1, 1, 24, 38, 512, 0, True, 512, False),
    ('conv', 1, 24, 38, 512, 512, 512, 512, 3, 1, 1, 1, 24, 38, 512, 1, True, 512, False),
    ('conv', 1, 24, 38, 64, 64, 512, 512, 3, 1, 1, 1, 24, 38, 0, -1, False, 512, False),
    ('conv', 1, 24, 38, 64, 64, 512, 512, 3, 1, 1, 1, 24, 38, 0, 1, True, 512, False),
    ('conv', 1, 304, 288, 128, 128, 128, 128, 3, 1, 1, 1, 304, 288, 0, -1, False, 128, False),
    ('conv', 1, 304, 288, 128, 128, 128, 128, 3, 1, 1, 1, 304, 288, 0, 1, False, 128, False),
    ('conv', 1, 304, 288, 128, 128, 128, 128, 3, 1, 1, 1, 304, 288, 128, -1, False, 128, False),
    ('conv', 1, 304, 288, 128, 128, 128, 128, 3, 1, 1, 1, 304, 288, 128, 1, False, 128, False),
    ('conv', 1, 304, 288, 128, 128, 128, 128, 3, 1, 1, 1, 304, 288, 128, 1, True, 128, False),
    ('conv', 1, 304, 288, 128, 128, 16, 16, 3, 1, 1, 1, 304, 288, 0, -1, False, 16, False),
    ('conv', 1, 304, 288, 256, 256, 128, 128, 1, 1, 0, 0, 304, 288, 0, -1, False, 128, False),
    ('conv', 1, 304, 288, 256, 256, 128, 128, 3, 1, 1, 1, 304, 288, 0, -1, False, 128, False),
    ('conv', 1, 304, 288, 256, 256, 128, 128, 3, 1, 1, 1, 304, 288, 0, 1, False, 128, False),
    ('conv', 1, 304, 304, 128, 128, 128, 128, 3, 1, 1, 1, 304, 304, 0, -1, False, 128, False),
    ('conv', 1, 304, 304, 128, 128, 128, 128, 3, 1, 1, 1, 304, 304, 0, 1, False, 128, False),
    ('conv', 1, 304, 304, 128, 128, 128, 128, 3, 1, 1, 1, 304, 304, 128, -1, False, 128, False),
    ('conv', 1, 304, 304, 128, 128, 128, 128, 3, 1, 1, 1, 304, 304, 128, 1, False, 128, False),
    ('conv', 1, 304, 304, 128, 128, 128, 128, 3, 1, 1, 1, 304, 304, 128, 1, True, 128, False),
    ('conv', 1, 304, 304, 128, 128, 16, 16, 3, 1, 1, 1, 304, 304, 0, -1, False, 16, False),
    ('conv', 1, 304, 304, 256, 256, 128, 128, 1, 1, 0, 0, 304, 304, 0, -1, False, 128, False),
    ('conv', 1, 304, 304, 256, 256, 128, 128, 3, 1, 1, 1, 304, 304, 0, -1, False, 128, False),
    ('conv', 1, 304, 304, 256, 256, 128, 128, 3, 1, 1, 1, 304, 304, 0, 1, False, 128, False),
    ('conv', 1, 32, 18, 256, 256, 512, 512, 1, 1, 0, 0, 32, 18, 0, -1, False, 512, False),
    ('conv', 1, 32, 18, 256, 256, 512, 512, 3, 1, 1, 1, 32, 18, 0, -1, False, 512, False),
    ('conv', 1, 32, 18, 256, 256, 512, 512, 3, 1, 1, 1, 32, 18, 0, 1, False, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 1, 1, 1, 32, 18, 0, -1, False, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 1, 1, 1, 32, 18, 0, 1, False, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 1, 1, 1, 32, 18, 512, -1, False, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 1, 1, 1, 32, 18, 512, 1, True, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 2, 0, 0, 16, 9, 0, -1, False, 512, False),
    ('conv', 1, 32, 18, 512, 512, 512, 512, 3, 2, 0, 0, 16, 9, 0, 1, True, 512, False),
    ('conv', 1, 32, 32, 256, 256, 512, 512, 1, 1, 0, 0, 32, 32, 0, -1, False, 512, False),
    ('conv', 1, 32, 32, 256, 256, 512, 512, 3, 1, 1, 1, 32, 32, 0, -1, False, 512, False),
    ('conv', 1, 32, 32, 256, 256, 512, 512, 3, 1, 1, 1, 32, 32, 0, 1, False, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 1, 1, 1, 32, 32, 0, -1, False, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 1, 1, 1, 32, 32, 0, 1, False, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 1, 1, 1, 32, 32, 512, -1, False, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 1, 1, 1, 32, 32, 512, 1, True, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 2, 0, 0, 16, 16, 0, -1, False, 512, False),
    ('conv', 1, 32, 32, 512, 512, 512, 512, 3, 2, 0, 0, 16, 16, 0, 1, True, 512, False),
    ('conv', 1, 36, 36, 128, 128, 256, 256, 1, 1, 0, 0, 36, 36, 0, -1, False, 256, False),
    ('conv', 1, 36, 36, 128, 128, 256, 256, 3, 1, 1, 1, 36, 36, 0, -1, False, 256, False),
    ('conv', 1, 36, 36, 128, 128, 256, 256, 3, 1, 1, 1, 36, 36, 0, 1, False, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 1, 1, 1, 36, 36, 0, -1, False, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 1, 1, 1, 36, 36, 0, 1, False, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 1, 1, 1, 36, 36, 256, -1, False, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 1, 1, 1, 36, 36, 256, 1, True, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 2, 0, 0, 18, 18, 0, -1, False, 256, False),
    ('conv', 1, 36, 36, 256, 256, 256, 256, 3, 2, 0, 0, 18, 18, 0, 1, True, 256, False),
    ('conv', 1, 36, 64, 128, 128, 256, 256, 1, 1, 0, 0, 36, 64, 0, -1, False, 256, False),
    ('conv', 1, 36, 64, 128, 128, 256, 256, 3, 1, 1, 1, 36, 64, 0, -1, False, 256, False),
    ('conv', 1, 36, 64, 128, 128, 256, 256, 3, 1, 1, 1, 36, 64, 0, 1, False, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 1, 1, 1, 36, 64, 0, -1, False, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 1, 1, 1, 36, 64, 0, 1, False, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 1, 1, 1, 36, 64, 256, -1, False, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 1, 1, 1, 36, 64, 256, 1, True, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 2, 0, 0, 18, 32, 0, -1, False, 256, False),
    ('conv', 1, 36, 64, 256, 256, 256, 256, 3, 2, 0, 0, 18, 32, 0, 1, True, 256, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 1, 1, 0, 0, 38, 36, 512, -1, False, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 1, 1, 0, 0, 38, 36, 512, 1, True, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 3, 1, 1, 1, 38, 36, 0, -1, False, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 3, 1, 1, 1, 38, 36, 0, 1, False, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 3, 1, 1, 1, 38, 36, 512, -1, False, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 3, 1, 1, 1, 38, 36, 512, 0, True, 512, False),
    ('conv', 1, 38, 36, 512, 512, 512, 512, 3, 1, 1, 1, 38, 36, 512, 1, True, 512, False),
    ('conv', 1, 38, 36, 64, 64, 512, 512, 3, 1, 1, 1, 38, 36, 0, -1, False, 512, False),
    ('conv', 1, 38, 36, 64, 64, 512, 512, 3, 1, 1, 1, 38, 36, 0, 1, True, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 1, 1, 0, 0, 38, 38, 512, -1, False, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 1, 1, 0, 0, 38, 38, 512, 1, True, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 3, 1, 1, 1, 38, 38, 0, -1, False, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 3, 1, 1, 1, 38, 38, 0, 1, False, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 3, 1, 1, 1, 38, 38, 512, -1, False, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 3, 1, 1, 1, 38, 38, 512, 0, True, 512, False),
    ('conv', 1, 38, 38, 512, 512, 512, 512, 3, 1, 1, 1, 38, 38, 512, 1, True, 512, False),
    ('conv', 1, 38, 38, 64, 64, 512, 512, 3, 1, 1, 1, 38, 38, 0, -1, False, 512, False),
    ('conv', 1, 38, 38, 64, 64, 512, 512, 3, 1, 1, 1, 38, 38, 0, 1, True, 512, False),
    ('conv', 1, 48, 64, 128, 128, 128, 128, 3, 1, 1, 1, 48, 64, 0, -1, False, 128, False),
    ('conv', 1, 48, 64, 128, 128, 128, 128, 3, 1, 1, 1, 48, 64, 128, -1, False, 128, False),
    ('conv', 1, 48, 64, 128, 128, 128, 128, 3, 2, 0, 0, 24, 32, 0, -1, False, 128, False),
    ('conv', 1, 48, 64, 256, 256, 256, 256, 3, 1, 1, 1, 48, 64, 0, -1, False, 256, False),
    ('conv', 1, 48, 64, 256, 256, 256, 256, 3, 1, 1, 1, 48, 64, 256, -1, False, 256, False),
    ('conv', 1, 48, 64, 512, 512, 256, 256, 1, 1, 0, 0, 48, 64, 0, -1, False, 256, False),
    ('conv', 1, 48, 64, 512, 512, 256, 256, 3, 1, 1, 1, 48, 64, 0, -1, False, 256, False),
    ('conv', 1, 48, 64, 64, 64, 128, 128, 3, 1, 1, 1, 48, 64, 0, -1, False, 128, False),
    ('conv', 1, 48, 72, 512, 512, 512, 512, 3, 1, 1, 1, 48, 72, 0, -1, False, 512, False),
    ('conv', 1, 48, 72, 512, 512, 512, 512, 3, 1, 1, 1, 48, 72, 0, 1, False, 512, False),
    ('conv', 1, 48, 72, 512, 512, 512, 512, 3, 1, 1, 1, 48, 72, 512, -1, False, 512, False),
    ('conv', 1, 48, 72, 512, 512, 512, 512, 3, 1, 1, 1, 48, 72, 512, 1, True, 512, False),
    ('conv', 1, 48, 76, 512, 512, 512, 512, 3, 1, 1, 1, 48, 76, 0, -1, False, 512, False),
    ('conv', 1, 48, 76, 512, 512, 512, 512, 3, 1, 1, 1, 48, 76, 0, 1, False, 512, False),
    ('conv', 1, 48, 76, 512, 512, 512, 512, 3, 1, 1, 1, 48, 76, 512, -1, False, 512, False),
    ('conv', 1, 48, 76, 512, 512, 512, 512, 3, 1, 1, 1, 48, 76, 512, 1, True, 512, False),
    ('conv', 1, 6, 8, 512, 512, 512, 512, 1, 1, 0, 0, 6, 8, 512, -1, False, 512, False),
    ('conv', 1, 6, 8, 512, 512, 512, 512, 3, 1, 1, 1, 6, 8, 0, -1, False, 512, False),
    ('conv', 1, 6, 8, 512, 512, 512, 512, 3, 1, 1, 1, 6, 8, 512, -1, False, 512, False),
    ('conv', 1, 64, 36, 128, 128, 256, 256, 1, 1, 0, 0, 64, 36, 0, -1, False, 256, False),
    ('conv', 1, 64, 36, 128, 128, 256, 256, 3, 1, 1, 1, 64, 36, 0, -1, False, 256, False),
    ('conv', 1, 64, 36, 128, 128, 256, 256, 3, 1, 1, 1, 64, 36, 0, 1, False, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 1, 1, 1, 64, 36, 0, -1, False, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 1, 1, 1, 64, 36, 0, 1, False, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 1, 1, 1, 64, 36, 256, -1, False, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 1, 1, 1, 64, 36, 256, 1, True, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 2, 0, 0, 32, 18, 0, -1, False, 256, False),
    ('conv', 1, 64, 36, 256, 256, 256, 256, 3, 2, 0, 0, 32, 18, 0, 1, True, 256, False),
    ('conv', 1, 64, 64, 128, 128, 256, 256, 1, 1, 0, 0, 64, 64, 0, -1, False, 256, False),
    ('conv', 1, 64, 64, 128, 128, 256, 256, 3, 1, 1, 1, 64, 64, 0, -1, False, 256, False),
    ('conv', 1, 64, 64, 128, 128, 256, 256, 3, 1, 1, 1, 64, 64, 0, 1, False, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, 1, 64, 64, 0, -1, False, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, 1, 64, 64, 0, 1, False, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, 1, 64, 64, 256, -1, False, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, 1, 64, 64, 256, 1, True, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 2, 0, 0, 32, 32, 0, -1, False, 256, False),
    ('conv', 1, 64, 64, 256, 256, 256, 256, 3, 2, 0, 0, 32, 32, 0, 1, True, 256, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 1, 1, 1, 72, 128, 0, -1, False, 128, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 1, 1, 1, 72, 128, 0, 1, False, 128, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 1, 1, 1, 72, 128, 128, -1, False, 128, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 1, 1, 1, 72, 128, 128, 1, True, 128, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 2, 0, 0, 36, 64, 0, -1, False, 128, False),
    ('conv', 1, 72, 128, 128, 128, 128, 128, 3, 2, 0, 0, 36, 64, 0, 1, True, 128, False),
    ('conv', 1, 72, 128, 64, 64, 128, 128, 3, 1, 1, 1, 72, 128, 0, -1, False, 128, False),
    ('conv', 1, 72, 128, 64, 64, 128, 128, 3, 1, 1, 1, 72, 128, 0, 1, True, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 1, 1, 1, 72, 72, 0, -1, False, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 1, 1, 1, 72, 72, 0, 1, False, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 1, 1, 1, 72, 72, 128, -1, False, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 1, 1, 1, 72, 72, 128, 1, True, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 2, 0, 0, 36, 36, 0, -1, False, 128, False),
    ('conv', 1, 72, 72, 128, 128, 128, 128, 3, 2, 0, 0, 36, 36, 0, 1, True, 128, False),
    ('conv', 1, 72, 72, 64, 64, 128, 128, 3, 1, 1, 1, 72, 72, 0, -1, False, 128, False),
    ('conv', 1, 72, 72, 64, 64, 128, 128, 3, 1, 1, 1, 72, 72, 0, 1, True, 128, False),
    ('conv', 1, 76, 72, 512, 512, 512, 512, 3, 1, 1, 1, 76, 72, 0, -1, False, 512, False),
    ('conv', 1, 76, 72, 512, 512, 512, 512, 3, 1, 1, 1, 76, 72, 0, 1, False, 512, False),
    ('conv', 1, 76, 72, 512, 512, 512, 512, 3, 1, 1, 1, 76, 72, 512, -1, False, 512, False),
    ('conv', 1, 76, 72, 512, 512, 512, 512, 3, 1, 1, 1, 76, 72, 512, 1, True, 512, False),
    ('conv', 1, 76, 76, 512, 512, 512, 512, 3, 1, 1, 1, 76, 76, 0, -1, False, 512, False),
    ('conv', 1, 76, 76, 512, 512, 512, 512, 3, 1, 1, 1, 76, 76, 0, 1, False, 512, False),
    ('conv', 1, 76, 76, 512, 512, 512, 512, 3, 1, 1, 1, 76, 76, 512, -1, False, 512, False),
    ('conv', 1, 76, 76, 512, 512, 512, 512, 3, 1, 1, 1, 76, 76, 512, 1, True, 512, False),
    ('conv', 1, 9, 16, 512, 512, 16, 16, 3, 1, 1, 1, 9, 16, 0, -1, False, 16, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 1, 1, 0, 0, 9, 16, 512, -1, False, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 1, 1, 0, 0, 9, 16, 512, 1, True, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 0, -1, False, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 0, 1, False, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 512, -1, False, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 512, 0, True, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 512, 1, False, 512, False),
    ('conv', 1, 9, 16, 512, 512, 512, 512, 3, 1, 1, 1, 9, 16, 512, 1, True, 512, False),
    ('conv', 1, 9, 9, 512, 512, 16, 16, 3, 1, 1, 1, 9, 9, 0, -1, False, 16, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 1, 1, 0, 0, 9, 9, 512, -1, False, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 1, 1, 0, 0, 9, 9, 512, 1, True, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 0, -1, False, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 0, 1, False, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 512, -1, False, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 512, 0, True, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 512, 1, False, 512, False),
    ('conv', 1, 9, 9, 512, 512, 512, 512, 3, 1, 1, 1, 9, 9, 512, 1, True, 512, False),
    ('conv', 1, 96, 128, 128, 128, 128, 128, 3, 1, 1, 1, 96, 128, 0, -1, False, 128, False),
    ('conv', 1, 96, 128, 128, 128, 128, 128, 3, 1, 1, 1, 96, 128, 128, -1, False, 128, False),
    ('conv', 1, 96, 128, 256, 256, 128, 128, 1, 1, 0, 0, 96, 128, 0, -1, False, 128, False),
    ('conv', 1, 96, 128, 256, 256, 128, 128, 3, 1, 1, 1, 96, 128, 0, -1, False, 128, False),
    ('conv', 1, 96, 144, 256, 256, 256, 256, 3, 1, 1, 1, 96, 144, 0, -1, False, 256, False),
    ('conv', 1, 96, 144, 256, 256, 256, 256, 3, 1, 1, 1, 96, 144, 0, 1, False, 256, False),
    ('conv', 1, 96, 144, 256, 256, 256, 256, 3, 1, 1, 1, 96, 144, 256, -1, False, 256, False),
    ('conv', 1, 96, 144, 256, 256, 256, 256, 3, 1, 1, 1, 96, 144, 256, 1, True, 256, False),
    ('conv', 1, 96, 144, 512, 512, 256, 256, 1, 1, 0, 0, 96, 144, 0, -1, False, 256, False),
    ('conv', 1, 96, 144, 512, 512, 256, 256, 3, 1, 1, 1, 96, 144, 0, -1, False, 256, False),
    ('conv', 1, 96, 144, 512, 512, 256, 256, 3, 1, 1, 1, 96, 144, 0, 1, False, 256, False),
    ('conv', 1, 96, 152, 256, 256, 256, 256, 3, 1, 1, 1, 96, 152, 0, -1, False, 256, False),
    ('conv', 1, 96, 152, 256, 256, 256, 256, 3, 1, 1, 1, 96, 152, 0, 1, False, 256, False),
    ('conv', 1, 96, 152, 256, 256, 256, 256, 3, 1, 1, 1, 96, 152, 256, -1, False, 256, False),
    ('conv', 1, 96, 152, 256, 256, 256, 256, 3, 1, 1, 1, 96, 152, 256, 1, True, 256, False),
    ('conv', 1, 96, 152, 512, 512, 256, 256, 1, 1, 0, 0, 96, 152, 0, -1, False, 256, False),
    ('conv', 1, 96, 152, 512, 512, 256, 256, 3, 1, 1, 1, 96, 152, 0, -1, False, 256, False),
    ('conv', 1, 96, 152, 512, 512, 256, 256, 3, 1, 1, 1, 96, 152, 0, 1, False, 256, False),
    ('gemm', 1368, 1368, 1368, 512, 512, 1368, 512, 1.0, False, False),
    ('gemm', 1368, 512, 512, 1368, 1368, 512, 1368, 0.04419417382415922, False, False),
    ('gemm', 1368, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 144, 144, 144, 512, 512, 144, 512, 1.0, False, False),
    ('gemm', 144, 512, 512, 144, 144, 512, 144, 0.04419417382415922, False, False),
    ('gemm', 144, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 1444, 1448, 1448, 512, 512, 1448, 512, 1.0, False, False),
    ('gemm', 1444, 512, 512, 1444, 1444, 512, 1448, 0.04419417382415922, False, False),
    ('gemm', 1444, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 192, 192, 192, 512, 512, 192, 512, 1.0, False, False),
    ('gemm', 192, 512, 512, 192, 192, 512, 192, 0.04419417382415922, False, False),
    ('gemm', 192, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 256, 256, 256, 512, 512, 256, 512, 1.0, False, False),
    ('gemm', 256, 512, 512, 256, 256, 512, 256, 0.04419417382415922, False, False),
    ('gemm', 256, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 48, 48, 48, 512, 512, 48, 512, 1.0, False, False),
    ('gemm', 48, 512, 512, 48, 48, 512, 48, 0.04419417382415922, False, False),
    ('gemm', 48, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 512, 512, 512, 1368, 1368, 512, 1368, 1.0, True, True),
    ('gemm', 512, 512, 512, 144, 144, 512, 144, 1.0, True, True),
    ('gemm', 512, 512, 512, 1444, 1444, 512, 1448, 1.0, True, True),
    ('gemm', 512, 512, 512, 192, 192, 512, 192, 1.0, True, True),
    ('gemm', 512, 512, 512, 256, 256, 512, 256, 1.0, True, True),
    ('gemm', 512, 512, 512, 48, 48, 512, 48, 1.0, True, True),
    ('gemm', 512, 512, 512, 81, 81, 512, 88, 1.0, True, True),
    ('gemm', 512, 512, 512, 864, 864, 512, 864, 1.0, True, True),
    ('gemm', 512, 512, 512, 912, 912, 512, 912, 1.0, True, True),
    ('gemm', 81, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 81, 512, 512, 81, 81, 512, 88, 0.04419417382415922, False, False),
    ('gemm', 81, 88, 88, 512, 512, 88, 512, 1.0, False, False),
    ('gemm', 864, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 864, 512, 512, 864, 864, 512, 864, 0.04419417382415922, False, False),
    ('gemm', 864, 864, 864, 512, 512, 864, 512, 1.0, False, False),
    ('gemm', 912, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 912, 512, 512, 912, 912, 512, 912, 0.04419417382415922, False, False),
    ('gemm', 912, 912, 912, 512, 512, 912, 512, 1.0, False, False),
    ('gn_apply', 12, 16, 256, True, True, True),
    ('gn_apply', 12, 16, 512, True, True, False),
    ('gn_apply', 12, 16, 512, True, True, True),
    ('gn_apply', 128, 128, 128, True, True, True),
    ('gn_apply', 128, 72, 128, True, True, True),
    ('gn_apply', 152, 144, 256, True, True, True),
    ('gn_apply', 152, 144, 512, True, True, True),
    ('gn_apply', 152, 152, 256, True, True, True),
    ('gn_apply', 152, 152, 512, True, True, True),
    ('gn_apply', 16, 16, 512, True, True, False),
    ('gn_apply', 16, 16, 512, True, True, True),
    ('gn_apply', 16, 9, 512, True, True, False),
    ('gn_apply', 16, 9, 512, True, True, True),
    ('gn_apply', 18, 18, 256, True, True, True),
    ('gn_apply', 18, 18, 512, True, True, True),
    ('gn_apply', 18, 32, 256, True, True, True),
    ('gn_apply', 18, 32, 512, True, True, True),
    ('gn_apply', 192, 288, 128, True, True, True),
    ('gn_apply', 192, 288, 256, True, True, True),
    ('gn_apply', 192, 304, 128, True, True, True),
    ('gn_apply', 192, 304, 256, True, True, True),
    ('gn_apply', 24, 32, 128, True, True, True),
    ('gn_apply', 24, 32, 256, True, True, True),
    ('gn_apply', 24, 32, 512, True, True, True),
    ('gn_apply', 24, 36, 512, True, True, False),
    ('gn_apply', 24, 36, 512, True, True, True),
    ('gn_apply', 24, 38, 512, True, True, False),
    ('gn_apply', 24, 38, 512, True, True, True),
    ('gn_apply', 304, 288, 128, True, True, True),
    ('gn_apply', 304, 288, 256, True, True, True),
    ('gn_apply', 304, 304, 128, True, True, True),
    ('gn_apply', 304, 304, 256, True, True, True),
    ('gn_apply', 32, 18, 256, True, True, True),
    ('gn_apply', 32, 18, 512, True, True, True),
    ('gn_apply', 32, 32, 256, True, True, True),
    ('gn_apply', 32, 32, 512, True, True, True),
    ('gn_apply', 36, 36, 128, True, True, True),
    ('gn_apply', 36, 36, 256, True, True, True),
    ('gn_apply', 36, 64, 128, True, True, True),
    ('gn_apply', 36, 64, 256, True, True, True),
    ('gn_apply', 38, 36, 512, True, True, False),
    ('gn_apply', 38, 36, 512, True, True, True),
    ('gn_apply', 38, 38, 512, True, True, False),
    ('gn_apply', 38, 38, 512, True, True, True),
    ('gn_apply', 48, 64, 128, True, True, True),
    ('gn_apply', 48, 64, 256, True, True, True),
    ('gn_apply', 48, 64, 512, True, True, True),
    ('gn_apply', 48, 72, 512, True, True, True),
    ('gn_apply', 48, 76, 512, True, True, True),
    ('gn_apply', 6, 8, 512, True, True, False),
    ('gn_apply', 6, 8, 512, True, True, True),
    ('gn_apply', 64, 36, 128, True, True, True),
    ('gn_apply', 64, 36, 256, True, True, True),
    ('gn_apply', 64, 64, 128, True, True, True),
    ('gn_apply', 64, 64, 256, True, True, True),
    ('gn_apply', 72, 128, 128, True, True, True),
    ('gn_apply', 72, 72, 128, True, True, True),
    ('gn_apply', 76, 72, 512, True, True, True),
    ('gn_apply', 76, 76, 512, True, True, True),
    ('gn_apply', 9, 16, 512, True, True, False),
    ('gn_apply', 9, 16, 512, True, True, True),
    ('gn_apply', 9, 9, 512, True, True, False),
    ('gn_apply', 9, 9, 512, True, True, True),
    ('gn_apply', 96, 128, 128, True, True, True),
    ('gn_apply', 96, 128, 256, True, True, True),
    ('gn_apply', 96, 144, 256, True, True, True),
    ('gn_apply', 96, 144, 512, True, True, True),
    ('gn_apply', 96, 152, 256, True, True, True),
    ('gn_apply', 96, 152, 512, True, True, True),
    ('gn_stats', 12, 16, 256, 32),
    ('gn_stats', 12, 16, 512, 32),
    ('gn_stats', 128, 128, 128, 32),
    ('gn_stats', 128, 72, 128, 32),
    ('gn_stats', 152, 144, 256, 32),
    ('gn_stats', 152, 144, 512, 32),
    ('gn_stats', 152, 152, 256, 32),
    ('gn_stats', 152, 152, 512, 32),
    ('gn_stats', 16, 16, 512, 32),
    ('gn_stats', 16, 9, 512, 32),
    ('gn_stats', 18, 18, 256, 32),
    ('gn_stats', 18, 18, 512, 32),
    ('gn_stats', 18, 32, 256, 32),
    ('gn_stats', 18, 32, 512, 32),
    ('gn_stats', 192, 288, 128, 32),
    ('gn_stats', 192, 288, 256, 32),
    ('gn_stats', 192, 304, 128, 32),
    ('gn_stats', 192, 304, 256, 32),
    ('gn_stats', 24, 32, 128, 32),
    ('gn_stats', 24, 32, 256, 32),
    ('gn_stats', 24, 32, 512, 32),
    ('gn_stats', 24, 36, 512, 32),
    ('gn_stats', 24, 38, 512, 32),
    ('gn_stats', 304, 288, 128, 32),
    ('gn_stats', 304, 288, 256, 32),
    ('gn_stats', 304, 304, 128, 32),
    ('gn_stats', 304, 304, 256, 32),
    ('gn_stats', 32, 18, 256, 32),
    ('gn_stats', 32, 18, 512, 32),
    ('gn_stats', 32, 32, 256, 32),
    ('gn_stats', 32, 32, 512, 32),
    ('gn_stats', 36, 36, 128, 32),
    ('gn_stats', 36, 36, 256, 32),
    ('gn_stats', 36, 64, 128, 32),
    ('gn_stats', 36, 64, 256, 32),
    ('gn_stats', 38, 36, 512, 32),
    ('gn_stats', 38, 38, 512, 32),
    ('gn_stats', 48, 64, 128, 32),
    ('gn_stats', 48, 64, 256, 32),
    ('gn_stats', 48, 64, 512, 32),
    ('gn_stats', 48, 72, 512, 32),
    ('gn_stats', 48, 76, 512, 32),
    ('gn_stats', 6, 8, 512, 32),
    ('gn_stats', 64, 36, 128, 32),
    ('gn_stats', 64, 36, 256, 32),
    ('gn_stats', 64, 64, 128, 32),
    ('gn_stats', 64, 64, 256, 32),
    ('gn_stats', 72, 128, 128, 32),
    ('gn_stats', 72, 72, 128, 32),
    ('gn_stats', 76, 72, 512, 32),
    ('gn_stats', 76, 76, 512, 32),
    ('gn_stats', 9, 16, 512, 32),
    ('gn_stats', 9, 9, 512, 32),
    ('gn_stats', 96, 128, 128, 32),
    ('gn_stats', 96, 128, 256, 32),
    ('gn_stats', 96, 144, 256, 32),
    ('gn_stats', 96, 144, 512, 32),
    ('gn_stats', 96, 152, 256, 32),
    ('gn_stats', 96, 152, 512, 32),
    ('softmax', 1368, 1368, 1368, True),
    ('softmax', 144, 144, 144, True),
    ('softmax', 1444, 1448, 1444, True),
    ('softmax', 192, 192, 192, True),
    ('softmax', 256, 256, 256, True),
    ('softmax', 48, 48, 48, True),
    ('softmax', 81, 88, 81, True),
    ('softmax', 864, 864, 864, True),
    ('softmax', 912, 912, 912, True),
    ('up2', 1, 12, 16, 512, 512, -1, False),
    ('up2', 1, 152, 144, 256, 256, -1, False),
    ('up2', 1, 152, 144, 256, 256, 1, True),
    ('up2', 1, 152, 152, 256, 256, -1, False),
    ('up2', 1, 152, 152, 256, 256, 1, True),
    ('up2', 1, 24, 32, 512, 512, -1, False),
    ('up2', 1, 24, 36, 512, 512, -1, False),
    ('up2', 1, 24, 36, 512, 512, 1, True),
    ('up2', 1, 24, 38, 512, 512, -1, False),
    ('up2', 1, 24, 38, 512, 512, 1, True),
    ('up2', 1, 38, 36, 512, 512, -1, False),
    ('up2', 1, 38, 36, 512, 512, 1, True),
    ('up2', 1, 38, 38, 512, 512, -1, False),
    ('up2', 1, 38, 38, 512, 512, 1, True),
    ('up2', 1, 48, 64, 256, 256, -1, False),
    ('up2', 1, 48, 72, 512, 512, -1, False),
    ('up2', 1, 48, 72, 512, 512, 1, True),
    ('up2', 1, 48, 76, 512, 512, -1, False),
    ('up2', 1, 48, 76, 512, 512, 1, True),
    ('up2', 1, 76, 72, 512, 512, -1, False),
    ('up2', 1, 76, 72, 512, 512, 1, True),
    ('up2', 1, 76, 76, 512, 512, -1, False),
    ('up2', 1, 76, 76, 512, 512, 1, True),
    ('up2', 1, 96, 144, 256, 256, -1, False),
    ('up2', 1, 96, 144, 256, 256, 1, True),
    ('up2', 1, 96, 152, 256, 256, -1, False),
    ('up2', 1, 96, 152, 256, 256, 1, True),
]


def _replay(sig, dt, seed):
    """Run one census signature on random data against float64 with the bounds above."""
    ops = _ops()
    kind = sig[0]
    if kind == "conv":
        _, N, H, W, Cin, xp, cout, rows, k, stride, pt, pl, oh, ow, rp, act, dual, yp, bpr = sig
        assert rows == cout and not bpr and (stride == 1 and (pt, pl) == (k // 2, k // 2) or stride == 2 and (pt, pl) == (0, 0))
        r = _conv_case(dt, N, H, W, Cin, cout, k, stride=stride, seed=seed, residual=rp > 0, post=None if act < 0 else bool(act), dual=dual,
                       x_extra=xp - Cin, y_extra=yp - cout, r_extra=max(rp - cout, 0))
        assert r[0].shape == (N, oh, ow, cout)
        _within(*r[:3], "conv" if act < 0 or dual else "conv+post", dt, repr(sig))
        if dual:
            _within(*r[3:], "conv+post", dt, repr(sig) + " (post)")
    elif kind == "up2":
        _, N, H, W, Cin, cout, act, dual = sig
        got, a, b, _ = _upconv_case(dt, N, H, W, Cin, cout, seed=seed, post=None if act < 0 else bool(act), dual=dual)
        if dual:
            _within(got[0], *a, "up2", dt, repr(sig))
            _within(got[1], *b, "up2+post", dt, repr(sig) + " (post)")
        else:
            _within(got, a, b, "up2" if act < 0 else "up2+post", dt, repr(sig))
    elif kind == "gemm":
        _, M, K, ap, n, brows, bp, yp, alpha, has_bias, bpr = sig
        got, ref, bound, obuf, _ = _gemm_case(dt, M, K, n, seed=seed, a_pitch=ap, b_rows=brows, b_pitch=bp, y_pitch=yp, alpha=alpha,
                                              bias=has_bias, bias_per_row=bpr)
        _within(got, ref, bound, "gemm", dt, repr(sig))
        mask = torch.zeros(obuf.shape, dtype=torch.bool, device="cuda")
        mask[:M, :n] = True
        _assert_nan_kept(obuf, mask, repr(sig))
    elif kind == "attn":
        _, T, C, *_rest, alpha = sig
        q, k, v = _qkv(T, C, dt, seed)
        ref, bound = _attention64(q, k, v, alpha, dt)
        _within(ops.attention(q, k, v, alpha), ref, bound, "attention", dt, repr(sig))
    elif kind == "softmax":
        _, rows, pitch, cols, inplace = sig
        x = _randn((rows, pitch), seed, 3.0).to(dt)
        ref, bound = _softmax64(x, cols, dt)
        y = ops.softmax_rows(x.clone(), cols)
        if inplace:
            x2 = x.clone()
            assert torch.equal(ops.softmax_rows(x2, cols, out=x2), y)
        _within(y[:, :cols], ref, bound, "softmax", dt, repr(sig))
        assert not y[:, cols:].any()
    elif kind == "gn_stats":
        _, H, W, C, groups = sig
        _gn_stats_check(_randn((1, H, W, C), seed, 1.3, 0.8).to(dt), groups, dt, repr(sig))
    elif kind == "gn_apply":
        _, H, W, C, has_g, has_b, act = sig
        _gn_apply_check(_randn((1, H, W, C), seed, 1.3, 0.8).to(dt), has_g, has_b, act, dt, seed, repr(sig))
    elif kind == "up_nn":
        x = _randn(sig[1:], seed).to(dt)
        assert torch.equal(ops.upsample2x_nhwc(x), x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    else:
        raise AssertionError(f"unknown census entry {sig!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_census_signatures_against_float64(dn):
    dt = DTS[dn]
    for i, sig in enumerate(CENSUS):
        _replay(sig, dt, 1000 + 17 * i)


@pytest.mark.gpu
def test_census_is_complete():
    """Re-run the spy: every signature the engine issues today is in the committed census, so an engine change that
    adds a layer shape or call form cannot go untested."""
    seen = record_census()
    missing = [s for s in seen if s not in set(CENSUS)]
    assert not missing, f"{len(missing)} signatures missing from CENSUS, e.g. {missing[:5]}"
    print(f"census: {len(seen)} signatures seen, {len(CENSUS)} committed")
    convs = [s for s in CENSUS if s[0] == "conv" and s[2] > 1]
    assert any(s[13] < 16 for s in convs) and any(s[13] >= 16 for s in convs), "both pixel-tile shapes of images"


# ------------------------------------------------------------------------------------------------ 4. edge cases
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_nan_padding_is_never_read_or_written(dn):
    """NaN in every padding column of x, w and the residual past Cin / Cout, in the output's padding columns and in
    guard pixels past the last one: the result is within the bound and the poisoned output stays untouched.  Cin = 96
    and K = 200 leave a partial last 64-channel chunk (the TMA unit zero-fills it)."""
    dt = DTS[dn]
    ops = _ops()
    N, H, W, Cin, Cout = 1, 19, 27, 96, 48
    x = _pitched(_randn((N, H, W, Cin), 31, 0.7).to(dt), 16)
    w = _pitched(_randn((9, Cout, Cin), 32, (Cin * 9) ** -0.5).to(dt), 8)
    bias = _randn((Cout,), 33, 0.3)
    res = _pitched(_randn((N, H, W, Cout), 34, 0.5).to(dt), 8)
    yp, guard = 64, 37
    obuf = torch.full((N * H * W + guard, yp), float("nan"), dtype=dt, device="cuda")
    out = obuf[:N * H * W].view(N, H, W, yp)[..., :Cout]
    ops.conv2d_nhwc(x, w, bias, ksize=3, pad=(1, 1), residual=res, out=out)
    ref, mag = _conv64(x, w, 3, 1, (1, 1), H, W, Cout)
    v, e = _pre(ref, mag, 9 * Cin, 1.0, bias.double(), res)
    _within(out, v, _out_bound(v, e, dt), "conv", dt, f"NaN-poisoned conv {dn}")
    mask = torch.zeros(obuf.shape, dtype=torch.bool, device="cuda")
    mask[:N * H * W, :Cout] = True
    _assert_nan_kept(obuf, mask, "conv")
    # the GEMM with K = Tp = 200 (Tp % 64 = 8), wider pitches and 128 guard rows past M
    got, ref, bound, obuf, M = _gemm_case(dt, 300, 200, 72, seed=35, a_pitch=256, b_pitch=264, y_pitch=88, bias_per_row=True, guard=128)
    _within(got, ref, bound, "gemm", dt, f"NaN-poisoned GEMM {dn}")
    mask = torch.zeros(obuf.shape, dtype=torch.bool, device="cuda")
    mask[:M, :72] = True
    _assert_nan_kept(obuf, mask, "gemm")


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("cout", [3, 17, 33, 129])
def test_odd_cout_with_wider_output_pitch(dn, cout):
    """Odd Cout: the last channel takes store_pair's single-element branch and the next (padding) column is left alone."""
    dt = DTS[dn]
    extra = (cout + 7) // 8 * 8 + 8 - cout          # pitch: the next multiple of 8 plus one more 8-column group
    got, ref, bound = _conv_case(dt, 1, 23, 37, 64, cout, 3, seed=40 + cout, residual=True, r_extra=extra, y_extra=extra)
    _within(got, ref, bound, "conv", dt, f"Cout {cout}")
    buf = got.as_strided((1, 23, 37, got.stride(2)), got.stride())
    assert torch.isnan(buf[..., cout:].float()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("hw", [(7, 9), (1, 1), (11, 13)])
def test_vt_gemm_as_the_engine_issues_it(dn, hw):
    """V^T = Wv X^T + bv per row, written into vt[:, :T] of a [C, Tp] buffer (odd T: single-element stores), then
    P V^T with K = Tp, as TensorCoreBackend.attention's four-GEMM path."""
    dt = DTS[dn]
    ops = _ops()
    T, C = hw[0] * hw[1], 512
    Tp = ops.round_up(T, 8)
    x2 = _randn((T, C), 50, 0.7).to(dt)
    wv = _randn((C, C), 51, C ** -0.5).to(dt)
    bv = _randn((C,), 52, 0.3)
    vt = torch.full((C, Tp), float("nan"), dtype=dt, device="cuda")
    ops.gemm_nt(wv, x2, bias=bv, bias_per_row=True, out=vt[:, :T])
    ref = wv.double() @ x2.double().t()
    mag = wv.double().abs() @ x2.double().abs().t()
    v, e = _pre(ref, mag, C, 1.0, bv.double()[:, None])
    _within(vt[:, :T], v, _out_bound(v, e, dt), "gemm", dt, f"V^T T={T}")
    assert torch.isnan(vt[:, T:].float()).all(), "V^T GEMM wrote past T"
    vt[:, T:] = 0
    p = ops.softmax_rows(_randn((T, Tp), 53, 3.0).to(dt), T)
    o = ops.gemm_nt(p, vt)
    ref = p.double() @ vt.double().t()
    mag = p.double().abs() @ vt.double().abs().t()
    v, e = _pre(ref, mag, Tp, 1.0)
    _within(o, v, _out_bound(v, e, dt), "gemm", dt, f"P V^T T={T}")


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_dual_output_batch_of_two(dn):
    """dual with N = 2 for conv2d_nhwc and upconv2x_nhwc (the per-image y2 offset): both outputs bit-equal to the
    single-output calls and within their bounds."""
    dt = DTS[dn]
    ops = _ops()
    raw, rref, rb, normed, zref, zb = _conv_case(dt, 2, 17, 21, 128, 128, 3, seed=60, residual=True, post=True, dual=True)
    _within(raw, rref, rb, "conv", dt, "dual raw")
    _within(normed, zref, zb, "conv+post", dt, "dual post")
    got, (v, vb), (z, zb2), (x, w16, bias, pst) = _upconv_case(dt, 2, 9, 19, 64, 128, seed=61, post=True, dual=True)
    _within(got[0], v, vb, "up2", dt, "up2 dual raw")
    _within(got[1], z, zb2, "up2+post", dt, "up2 dual post")
    assert torch.equal(got[0], ops.upconv2x_nhwc(x, w16, bias))
    assert torch.equal(got[1], ops.upconv2x_nhwc(x, w16, bias, post=pst))
    for n in range(2):   # image n alone gives the same bits as image n of the batch
        one = ops.upconv2x_nhwc(x[n:n + 1].contiguous(), w16, bias, post=pst, dual=True)
        assert torch.equal(one[0][0], got[0][n]) and torch.equal(one[1][0], got[1][n])


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_dual_conv_batch_of_two_matches_single_output_calls(dn):
    dt = DTS[dn]
    ops = _ops()
    x = _randn((2, 17, 21, 128), 62, 0.7).to(dt)
    w = _randn((9, 128, 128), 63, (128 * 9) ** -0.5).to(dt)
    bias, res = _randn((128,), 64, 0.3), _randn((2, 17, 21, 128), 65, 0.5).to(dt)
    pst = (_randn((128,), 66, 0.4, 1.0), _randn((128,), 67, 0.2), True)
    raw, normed = ops.conv2d_nhwc(x, w, bias, ksize=3, pad=(1, 1), residual=res, post=pst, dual=True)
    assert torch.equal(raw, ops.conv2d_nhwc(x, w, bias, ksize=3, pad=(1, 1), residual=res))
    assert torch.equal(normed, ops.conv2d_nhwc(x, w, bias, ksize=3, pad=(1, 1), residual=res, post=pst))


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_silu_epilogue_at_large_magnitudes(dn):
    """Pre-activations around +-90: __expf(-t) overflows for t < -88.7 and __fdividef sees divisors above 2^126 for
    t < -87.3.  The outputs stay finite and within the bound (whose 2^-119 term covers the flush to 0)."""
    dt = DTS[dn]
    shifts = torch.tensor([-90.0, -88.5, -87.5, -87.0, -60.0, -20.0, 0.0, 20.0, 60.0, 87.5, 90.0, -89.0, -88.0, -86.0, -30.0, 30.0],
                          device="cuda").repeat(4)
    got, ref, bound = _conv_case(dt, 1, 12, 40, 64, 64, 1, seed=70, post=True, shift=shifts)
    _within(got, ref, bound, "conv+post", dt, "SiLU at +-90")


@pytest.mark.gpu
def test_conv_refuses_weights_with_more_rows_than_cout():
    """A 3x3 weight packed with more rows per tap than the Cout of the call would be read at the wrong tap offsets
    (the kernel steps taps by Cout rows): the wrapper refuses it.  A 1x1 weight (one tap) may carry extra rows."""
    ops = _ops()
    x = torch.zeros((1, 8, 8, 64), dtype=torch.float16, device="cuda")
    w = torch.zeros((9, 16, 64), dtype=torch.float16, device="cuda")
    with pytest.raises(AssertionError):
        ops.conv2d_nhwc(x, w, None, ksize=3, pad=(1, 1), cout=3)
    got = ops.conv2d_nhwc(x, w[:1].contiguous(), None, ksize=1, cout=8)
    assert got.shape == (1, 8, 8, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("T", [1, 7, 63, 64, 65, 129, 1000])
def test_fused_attention_short_sequences(dn, T):
    dt = DTS[dn]
    ops = _ops()
    C = 512
    q, k, v = _qkv(T, C, dt, 80 + T)
    q[0] = 0                       # a row whose logits are all equal: the uniform average of v
    alpha = C ** -0.5
    ref, bound = _attention64(q, k, v, alpha, dt)
    _within(ops.attention(q, k, v, alpha), ref, bound, "attention", dt, f"attention T={T}")


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_fused_attention_no_worse_than_four_gemm_path(dn):
    """At a small T the four-GEMM path (S rounded to 16 bits before the softmax) is the less accurate one."""
    dt = DTS[dn]
    ops = _ops()
    T, C = 65, 512
    q, k, v = _qkv(T, C, dt, 90)
    alpha = C ** -0.5
    Tp = ops.round_up(T, 8)
    vt = torch.zeros((C, Tp), dtype=dt, device="cuda")
    vt[:, :T] = v.T
    s = torch.empty((T, Tp), dtype=dt, device="cuda")
    ops.gemm_nt(q, k, alpha=alpha, out=s[:, :T])
    ops.softmax_rows(s, T, out=s)
    old = ops.gemm_nt(s, vt)
    new = ops.attention(q, k, v, alpha)
    ref, bound = _attention64(q, k, v, alpha, dt)
    _within(new, ref, bound, "attention", dt, "fused T=65")
    assert (new.double() - ref).abs().max() <= (old.double() - ref).abs().max()


SOFTMAX_CASES = [(5, 8, 1), (7, 16, 13), (3, 1008, 1003), (2, 72288, 72280)]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("rows,pitch,cols", SOFTMAX_CASES)
def test_softmax_rows_against_float64(dn, rows, pitch, cols):
    dt = DTS[dn]
    ops = _ops()
    x = torch.full((rows, pitch), 77.0, dtype=dt, device="cuda")
    x[:, :cols] = _randn((rows, cols), 100 + cols, 3.0).to(dt)
    ref, bound = _softmax64(x, cols, dt)
    y = ops.softmax_rows(x, cols)
    _within(y[:, :cols], ref, bound, "softmax", dt, f"softmax {rows}x{cols}/{pitch}")
    assert not y[:, cols:].any()
    x2 = x.clone()
    assert torch.equal(ops.softmax_rows(x2, cols, out=x2), y), "in-place differs from out-of-place"


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_softmax_rows_near_the_fp16_maximum(dn):
    dt = DTS[dn]
    ops = _ops()
    rows, cols, pitch = 4, 300, 304
    x = torch.zeros((rows, pitch), dtype=dt, device="cuda")
    x[:, :cols] = (65504.0 - _randn((rows, cols), 110, 4.0).abs()).to(dt)
    x[1, :cols:7] = torch.tensor(65504.0, dtype=dt) if dt == torch.float16 else torch.tensor(65280.0, dtype=dt)
    ref, bound = _softmax64(x, cols, dt)
    y = ops.softmax_rows(x, cols)
    _within(y[:, :cols], ref, bound, "softmax", dt, "softmax near 65504")
    x2 = x.clone()
    assert torch.equal(ops.softmax_rows(x2, cols, out=x2), y)


def _gn_stats_check(x, groups, dt, what, var_rtol=5e-5):
    """Tolerances of test_gpu_vae.py's statistics tests (mean rtol 2e-5 / atol 2e-6, var rtol 5e-5 / atol 1e-6;
    var rtol 2e-3 when mean >> std), against float64."""
    ops = _ops()
    var, mean = ops.gn_stats_nhwc(x, groups)
    C = x.shape[-1]
    xd = x.double().reshape(-1, groups, C // groups)
    wm = xd.mean(dim=(0, 2))
    wv = ((xd - wm[None, :, None]) ** 2).mean(dim=(0, 2))
    rm = ((mean.double() - wm).abs() / (2e-5 * wm.abs() + 2e-6)).max().item()
    rv = ((var.double() - wv).abs() / (var_rtol * wv.abs() + 1e-6)).max().item()
    _note("gn_stats", dt, max(rm, rv))
    assert (var >= 0).all(), f"{what}: negative variance"
    assert rm <= 1 and rv <= 1, f"{what}: mean err/tol {rm:.3g}, var err/tol {rv:.3g}"
    return var, mean


def _gn_apply_check(x, has_g, has_b, act, dt, seed, what):
    ops = _ops()
    C = x.shape[-1]
    mean = _randn((32,), seed + 1, 0.3, 0.8)
    var = _randn((32,), seed + 2, 0.2).abs() + 0.5
    gamma = _randn((C,), seed + 3, 0.5, 1.0) if has_g else None
    beta = _randn((C,), seed + 4, 0.2) if has_b else None
    got = ops.gn_apply_nhwc(x, mean, var, gamma, beta, act)
    ref, bound = _gn_apply64(x, mean, var, gamma, beta, act, dt)
    _within(got, ref, bound, "gn_apply", dt, what)


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
@pytest.mark.parametrize("C", [128, 256, 512])
def test_group_norm_nhwc_edges(dn, C):
    """Pixel counts below one CTA's pixels-per-iteration (256 / (C / 8)), a prime count and the census's largest
    tile; a constant input (variance exactly 0, never negative); mean >> std; gamma / beta as None."""
    dt = DTS[dn]
    largest = max((s[1] * s[2], s[1], s[2]) for s in CENSUS if s[0] == "gn_stats" and s[3] == C)[1:]
    for (h, w) in [(1, 3), (1, 1009), largest]:
        x = _randn((1, h, w, C), 120 + h + w, 1.3, 0.8).to(dt)
        var, mean = _gn_stats_check(x, 32, dt, f"stats {h}x{w}x{C}")
        for has_g, has_b, act in [(True, True, True), (True, True, False), (False, False, True), (False, True, False)]:
            _gn_apply_check(x, has_g, has_b, act, dt, 130, f"apply {h}x{w}x{C} {has_g} {has_b} {act}")
    const = torch.full((1, 33, 29, C), 1.75, dtype=dt, device="cuda")
    var, mean = _gn_stats_check(const, 32, dt, "constant")
    assert (var == 0).all() and (mean == 1.75).all()
    off = (_randn((1, 41, 37, C), 140, 0.01, 100.0)).to(dt)
    _gn_stats_check(off, 32, dt, "mean >> std", var_rtol=2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_wrap_gather_and_layout_kernels_bit_exact(dn):
    """nchw_to_nhwc_wrap with negative origins and tiles more than twice as wide / tall as the canvas == modular index
    arithmetic in torch; nhwc_to_nchw_region and upsample2x_nhwc with N = 2."""
    dt = DTS[dn]
    ops = _ops()
    z = _randn((2, 4, 7, 9), 150).to(dt)
    for bbox in [(-13, 20, -9, 12), (-1, 8, -20, -3), (5, 40, 3, 30)]:
        x1, x2, y1, y2 = bbox
        got = ops.nchw_to_nhwc_wrap(z, bbox, 64)
        ry = torch.arange(y1, y2, device="cuda") % 7
        rx = torch.arange(x1, x2, device="cuda") % 9
        want = z[:, :, ry][:, :, :, rx].permute(0, 2, 3, 1)
        assert torch.equal(got[..., :4], want), bbox
        assert not got[..., 4:].any()
    x = _randn((2, 13, 17, 24), 151).to(dt)
    dst = torch.full((2, 5, 30, 40), 3.0, dtype=dt, device="cuda")
    before = dst.clone()
    ops.nhwc_to_nchw_region(x[:, 2:11, 3:15, :], dst[:, :, 4:13, 6:18], 5)
    want = before.clone()
    want[:, :, 4:13, 6:18] = x[:, 2:11, 3:15, :5].permute(0, 3, 1, 2)
    assert torch.equal(dst, want)
    u = ops.upsample2x_nhwc(x.contiguous())
    assert torch.equal(u, x.repeat_interleave(2, 1).repeat_interleave(2, 2))


# ------------------------------------------------------------------------------------------------ 5. bf16 network end to end
# The fp16 bars of test_gpu_vae.py / test_gpu_attention.py scaled by the bf16 / fp16 unit-roundoff ratio (2^-8 / 2^-11 = 8):
# against the fp32 reference mean 2e-3 -> 1.6e-2, max 3e-2 -> 0.24; against the module backend on the same bf16
# network mean 1e-3 -> 8e-3, max 2e-2 -> 0.16 (all relative to max |reference|).
@pytest.mark.gpu
@pytest.mark.parametrize("is_dec,fast,H,W,tile", [(True, True, 40, 52, 16), (True, False, 40, 52, 16), (False, True, 200, 264, 64),
                                                  (False, False, 136, 200, 64)])
def test_bf16_network_matches_fp32_reference(is_dec, fast, H, W, tile):
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from oracle import synth, vae
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    z = synth.latent(5 if is_dec else 6, (1, 4 if is_dec else 3, H, W), torch.float32)
    with torch.no_grad():
        want = vae.vae_hook_call(_sd_width_net(is_dec, 3 if is_dec else 4).cuda(), z.cuda(), tile, is_dec, fast, False).cpu()
    net = _sd_width_net(is_dec, 3 if is_dec else 4).cuda().to(torch.bfloat16)
    hook = tilevae.VAEHook(net, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
    with torch.no_grad():
        got = hook(z.cuda().to(torch.bfloat16))
    assert hook.backend_name == "wgmma"
    assert got.dtype == torch.bfloat16 and got.shape == want.shape
    diff = (got.cpu().float() - want).abs()
    scale = want.abs().max().item()
    mean_r, max_r = diff.mean().item() / scale, diff.max().item() / scale
    print(f"bf16 {'decoder' if is_dec else 'encoder'} fast={fast} vs fp32: mean {mean_r:.3g}, max {max_r:.3g} of scale")
    assert mean_r <= 1.6e-2 and max_r <= 0.24, (mean_r, max_r)


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [True, False])
def test_bf16_tensor_core_backend_matches_module_backend(fast):
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    from oracle import synth
    net = _sd_width_net(True, 3).cuda().to(torch.bfloat16)
    z = synth.latent(5, (1, 4, 40, 52), torch.bfloat16).cuda()
    hook = tilevae.VAEHook(net, 16, True, fast, fast, False)
    with torch.no_grad():
        a = hook(z)
        assert hook.backend_name == "wgmma"
        orig = ve.pick_backend
        ve.pick_backend = lambda program, device, dtype: ve.ModuleBackend(program, device, dtype)
        try:
            b = hook(z)
        finally:
            ve.pick_backend = orig
    assert hook.backend_name == "modules"
    scale = b.float().abs().max().item()
    d = (a.float() - b.float()).abs()
    mean_r, max_r = d.mean().item() / scale, d.max().item() / scale
    print(f"bf16 decoder fast={fast} wgmma vs modules: mean {mean_r:.3g}, max {max_r:.3g} of scale")
    assert mean_r <= 8e-3 and max_r <= 0.16, (mean_r, max_r)


# ------------------------------------------------------------------------------------------------ 6. non-vacuity
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_bounds_catch_realistic_defects(dn):
    """The same comparisons against deliberately wrong float64 references must fail on some elements."""
    dt = DTS[dn]
    ops = _ops()
    found = {}
    # transposed 3x3 taps
    x = _randn((1, 18, 22, 64), 200, 0.7).to(dt)
    w = _randn((9, 64, 64), 201, (64 * 9) ** -0.5).to(dt)
    got = ops.conv2d_nhwc(x, w, None, ksize=3, pad=(1, 1))
    ref, mag = _conv64(x, w, 3, 1, (1, 1), 18, 22, 64)
    v, e = _pre(ref, mag, 9 * 64)
    assert _violations(got, v, _out_bound(v, e, dt)) == 0
    wt = w.view(3, 3, 64, 64).transpose(0, 1).reshape(9, 64, 64)
    r2, m2 = _conv64(x, wt, 3, 1, (1, 1), 18, 22, 64)
    v2, e2 = _pre(r2, m2, 9 * 64)
    found["transposed 3x3 taps"] = _violations(got, v2, _out_bound(v2, e2, dt))
    # output shifted by one pixel at the border (the last column repeats its neighbour)
    vs = v.clone()
    vs[:, :, -1] = v[:, :, -2]
    found["border pixel shifted"] = _violations(got, vs, _out_bound(vs, e, dt))
    # swapped up2 parities
    got, vv, b, (xu, w16, bias) = _upconv_case(dt, 1, 9, 11, 64, 64, seed=210)
    r3, m3 = _upconv64(xu, w16, 64, swap_parity=True)
    v3, e3 = _pre(r3, m3, 4 * 64, 1.0, bias.double())
    found["swapped up2 parities"] = _violations(got, v3, _out_bound(v3, e3, dt))
    # the last (partial) K chunk dropped: Cin = 96, channels 64..95 left out of the reference
    x = _randn((1, 15, 17, 96), 220, 0.7).to(dt)
    w = _randn((9, 32, 96), 221, (96 * 9) ** -0.5).to(dt)
    got = ops.conv2d_nhwc(x, w, None, ksize=3, pad=(1, 1))
    xc = x.clone()
    xc[..., 64:] = 0
    r4, m4 = _conv64(xc, w, 3, 1, (1, 1), 15, 17, 32)
    v4, e4 = _pre(r4, m4, 9 * 96)
    found["last K chunk dropped"] = _violations(got, v4, _out_bound(v4, e4, dt))
    # an online softmax that never rescales earlier key blocks
    q, k, vv = _qkv(1000, 512, dt, 230)
    got = ops.attention(q, k, vv, 512 ** -0.5)
    r5, b5 = _attention64(q, k, vv, 512 ** -0.5, dt, stale_max=True)
    found["P not renormalised"] = _violations(got, r5, b5)
    print(f"non-vacuity {dn}: " + ", ".join(f"{k_}: {n} elements fail" for k_, n in found.items()))
    assert all(n > 0 for n in found.values()), found


# ------------------------------------------------------------------------------------------------ 7. refusals (no GPU)
def _stream():
    return _cabi().current_stream_ptr() if torch.cuda.is_available() else None


def _scratch(nbytes=1 << 20):
    return torch.zeros(nbytes, dtype=torch.uint8, device="cuda" if torch.cuda.is_available() else "cpu")


def _desc(**over):
    """A valid 3x3 / stride 1 / pad 1 descriptor on 8 x 8 x 64 -> 64 fp16, with overrides."""
    cabi = _cabi()
    d = cabi.TdConvDesc(N=1, H=8, W=8, Cin=64, Cout=64, kh=3, kw=3, stride=1, pad_top=1, pad_left=1, OH=8, OW=8, dtype=cabi.TD_F16,
                        bias_per_row=0, alpha=1.0, x_pitch=64, w_pitch=64, y_pitch=64, res_pitch=0)
    for k_, v_ in over.items():
        setattr(d, k_, v_)
    return d


def _conv_call(buf, d, x_off=0, residual=False, up2=False):
    lib = _cabi().lib
    base = buf.data_ptr()
    x, w, y = base + x_off, base + (64 << 10), base + (256 << 10)
    if up2:
        return lib.td_upconv2x_nhwc(ctypes.byref(d), x, w, None, y, _stream())
    return lib.td_conv2d_nhwc(ctypes.byref(d), x, w, None, base + (512 << 10) if residual else None, y, _stream())


def test_conv_valid_descriptor_reaches_the_device():
    """The base descriptor of the refusal tests is accepted (without a device the device query then fails)."""
    cabi = _cabi()
    buf = _scratch()
    st = _conv_call(buf, _desc())
    assert st == (cabi.TD_OK if torch.cuda.is_available() else cabi.TD_ERR_CUDA), cabi.lib.td_last_error()
    st = _conv_call(buf, _desc(OH=16, OW=16), up2=True)
    assert st == (cabi.TD_OK if torch.cuda.is_available() else cabi.TD_ERR_CUDA), cabi.lib.td_last_error()
    if torch.cuda.is_available():
        torch.cuda.synchronize()


def _refusals(p):
    """(name, descriptor, call options, expected status); p: a device buffer for the second output / post vectors."""
    c = _cabi()
    return [
        ("Cin % 8", _desc(Cin=60), {}, c.TD_ERR_UNSUPPORTED),
        ("k = 5", _desc(kh=5, kw=5), {}, c.TD_ERR_UNSUPPORTED),
        ("stride 3", _desc(stride=3), {}, c.TD_ERR_UNSUPPORTED),
        ("fp32", _desc(dtype=c.TD_F32), {}, c.TD_ERR_UNSUPPORTED),
        ("x pitch < Cin", _desc(x_pitch=56), {}, c.TD_ERR_INVALID_ARG),
        ("y pitch < Cout", _desc(y_pitch=56), {}, c.TD_ERR_INVALID_ARG),
        ("residual pitch < Cout", _desc(res_pitch=56), {"residual": True}, c.TD_ERR_INVALID_ARG),
        ("misaligned x", _desc(), {"x_off": 2}, c.TD_ERR_INVALID_ARG),
        ("y2 without post", _desc(y2=p, y2_pitch=64), {}, c.TD_ERR_INVALID_ARG),
        ("post_scale without post_shift", _desc(post_scale=p), {}, c.TD_ERR_INVALID_ARG),
        ("up2 with bias per row", _desc(OH=16, OW=16, bias_per_row=1), {"up2": True}, c.TD_ERR_INVALID_ARG),
        ("up2 with OH != 2H", _desc(OH=15, OW=16), {"up2": True}, c.TD_ERR_INVALID_ARG),
        ("up2 with a 1x1 kernel", _desc(OH=16, OW=16, kh=1, kw=1), {"up2": True}, c.TD_ERR_INVALID_ARG),
    ]


def test_conv_refusals():
    """Each bad descriptor returns its status before any launch.  (td_upconv2x_nhwc has no residual argument: its
    descriptor's res_pitch is never used.)"""
    buf = _scratch()
    for name, d, kw, want in _refusals(buf.data_ptr() + (768 << 10)):
        st = _conv_call(buf, d, **kw)
        assert st == want, f"{name}: status {st} ({_cabi().lib.td_last_error().decode()})"


def test_nhwc_attention_softmax_refusals():
    cabi = _cabi()
    lib = cabi.lib
    buf = _scratch()
    p = buf.data_ptr()
    mean, var = p + (800 << 10), p + (900 << 10)
    # gn stats: C / 8 must divide 256 (C = 640 does not), and the workspace must hold one partial per CTA
    st = lib.td_gn_stats_nhwc(p, 100, 640, 32, cabi.TD_F16, p + (512 << 10), 1 << 16, mean, var, _stream())
    assert st == cabi.TD_ERR_UNSUPPORTED, lib.td_last_error()
    need = lib.td_gn_stats_nhwc_workspace_bytes(1000, 128, 32)
    assert need > 0
    st = lib.td_gn_stats_nhwc(p, 1000, 128, 32, cabi.TD_F16, p + (512 << 10), 1000, mean, var, _stream())
    assert st == cabi.TD_ERR_CAPACITY, lib.td_last_error()
    # softmax rows: pitch % 8 != 0
    st = lib.td_softmax_rows(p, p + (256 << 10), 2, 5, 12, cabi.TD_F16, _stream())
    assert st == cabi.TD_ERR_INVALID_ARG, lib.td_last_error()
    # attention: C = 576 > 512
    st = lib.td_attention(p, p, p, p + (512 << 10), 4, 576, 576, 576, 576, 576, 1.0, cabi.TD_F16, _stream())
    assert st == cabi.TD_ERR_UNSUPPORTED, lib.td_last_error()


# ------------------------------------------------------------------------------------------------ report
@pytest.mark.gpu
def test_zz_report_worst_ratios():
    """Prints the worst err / bound per op family and dtype seen by the tests above (run with -s)."""
    for (fam, dn), r in sorted(WORST.items()):
        print(f"worst err/bound {fam:10s} {dn:5s} {r:.3g}")
