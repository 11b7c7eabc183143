"""The tensor-core VAE kernels per element at the tile sizes an H100 runs: the reference's 80 GB defaults (decoder 256,
encoder 3072) and its UI maxima (decoder 512, encoder 4096), where single activations pass 2^31 bytes and 2^31
elements, GroupNorm groups pass 2^24 elements and the persistent convolution walks hundreds of thousands of pixel
tiles.  test_gpu_vae_kernels.py checks the same kernels at the small census shapes; its bounds are used here unchanged.

A float64 reference of a whole 4272 x 4272 x 128 convolution is out of reach, so the dense kernels are checked at a
sample of output pixels (all output channels of each): the first and last pixel, every pixel of the last (partial)
pixel tile in x, in y and of the corner tile, every pixel holding an element whose flat index crosses 2^30 or 2^31
(byte offsets 2^31 and 2^32) in y, y2 and the residual, and a few thousand seeded random pixels (`_sample_pixels`).
Each reference is computed in float64 on the GPU from the exact 16-bit inputs gathered at those pixels.  Fused
attention is checked at 256 query rows against all keys (`_attention_rows`).  The streaming kernels are checked over
the whole tensor, chunk by chunk.

gn_stats_nhwc bound.  A thread owns one 8-channel vector position and walks pixels p = slot + m G (G = grid * ppi
pixel slots, ppi = 256 / (C / 8), grid = min(ceil(P / ppi), 4 SMs)); each 4-channel half sums d = x - k, k the half's
first channel at the thread's first pixel, over n_t <= 4 ceil(P / G) elements.  The per-thread moments are merged with
Chan's update: serially over the CTA's ppi * cpg / 4 halves of the group, serially over ceil(grid / 32) partials per
lane of the final warp and through its 5 shuffle levels: depth D = ppi cpg / 4 + ceil(grid / 32) + 5.  This is the
structure the NCHW statistics bound of test_gpu_vae_nchw_kernels.py (`_stats_bounds`) covers, with S the sum of the
squared shifted values (computed here from the kernel's own shifts), except that the counts, which travel as float,
are not all exact: a group of more than 2^24 elements has partial counts past 2^26 whose float spacing (8) is coarser
than their granularity (4).  That adds at most one rounding to the count of each merge, so each merge carries one more
rounding in the mean (4 instead of 3) and two more in M2 (6 instead of 4).  That bound is worst case: at a
decoder-512 group (n_t = 8644, D = 38) it allows several times the variance, so the statistics must also meet the fixed
tolerances of test_gpu_vae_kernels._gn_stats_check (mean 2e-5 relative + 2e-6, variance 5e-5 relative + 1e-6).
"""
import time
import types

import pytest
import torch

from test_gpu_vae_kernels import (DN, DTS, _attention64, _gn_apply64, _out_bound, _post64, _pre, _sd_width_net, _softmax64, _within,
                                  census_spy, record_census)
from test_gpu_vae_nchw_kernels import STAT_THREADS, _apply64, _stats_bounds, plan_stats
from test_gpu_vae_nchw_kernels import _within as _within_nchw

GIB = 1 << 30
# flat element indices whose crossing is checked: 2^30 (a byte offset of 2^31 in 16 bits) and 2^31 (2^31 elements,
# a byte offset of 2^32)
CROSSINGS = (2 ** 30, 2 ** 31)
PEAK = {"bytes": 0, "base": 0}


def _ops():
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops
    return vae_ops


# ------------------------------------------------------------------------------------------------ memory and data
def _need(nbytes, what):
    """Fail (not skip) when the card cannot hold a case whose peak, computed from its shapes, is `nbytes`."""
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    assert free >= nbytes, (f"{what}: needs about {nbytes / 1e9:.1f} GB of device memory, but only {free / 1e9:.1f} GB of "
                            f"{total / 1e9:.1f} GB are free")


def _reset():
    """Start measuring a case: its peak is counted above what was already allocated (by other tests, too)."""
    torch.cuda.reset_peak_memory_stats()
    PEAK["base"] = torch.cuda.memory_allocated()


def _track():
    PEAK["bytes"] = max(PEAK["bytes"], torch.cuda.max_memory_allocated() - PEAK["base"])


def _fill(shape, seed, dt, scale=1.0, shift=0.0, chunk=1 << 27):
    """Seeded N(shift, scale^2) values rounded to dt, generated in chunks (no full-size fp32 temporary)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty(shape, dtype=dt, device="cuda")
    flat = out.view(-1)
    for s in range(0, flat.numel(), chunk):
        n = min(chunk, flat.numel() - s)
        flat[s:s + n] = (torch.randn(n, generator=g, device="cuda") * scale + shift).to(dt)
    return out


def _pitched_buf(rows, cols, pitch, dt, fill=float("nan"), guard=1):
    """[rows + guard, pitch] filled with `fill` (padding columns and `guard` rows past the end must keep it)."""
    return torch.full((rows + guard, pitch), fill, dtype=dt, device="cuda")


# ------------------------------------------------------------------------------------------------ sample positions
def _crossing_rows(pitch, rows):
    """Rows (pixels) of a [rows, pitch] buffer holding the elements on each side of every CROSSINGS index."""
    out = set()
    for e in CROSSINGS:
        for i in (e - 1, e):
            if i < rows * pitch:
                out.add(i // pitch)
    return out


def _last_tiles(OH, OW, BW, BH, up2):
    """Output pixels of the last pixel tile in x (first tile row), in y (first tile column) and of the corner tile, as
    td_conv2d_nhwc tiles its grid (up2: the low-resolution grid, once per output parity)."""
    gH, gW = (OH // 2, OW // 2) if up2 else (OH, OW)
    tx, ty = (gW - 1) // BW * BW, (gH - 1) // BH * BH
    out = set()
    for x0, y0 in {(tx, 0), (0, ty), (tx, ty)}:
        for y in range(y0, min(y0 + BH, gH)):
            for x in range(x0, min(x0 + BW, gW)):
                if up2:
                    out.update((2 * y + py) * OW + 2 * x + px for py in (0, 1) for px in (0, 1))
                else:
                    out.add(y * OW + x)
    return out


def _pixel_tile(OH, OW, up2):
    """td_conv2d_nhwc's pixel tile (BW, BH) for this output grid."""
    gH, gW = (OH // 2, OW // 2) if up2 else (OH, OW)
    if gH == 1:
        return 128, 1
    return (16, 8) if gW >= 16 else (8, 16)


def _sample_pixels(OH, OW, pitches, up2=False, n_random=3000, seed=0, gemm=False):
    """Sorted flat output pixels to check (see the module docstring); pitches: the pixel pitches (elements) of every
    tensor the kernel addresses per output pixel (y, y2, residual).  gemm: the rows of a GEMM (one pixel row)."""
    P = OH * OW
    BW, BH = (128, 1) if gemm else _pixel_tile(OH, OW, up2)
    pix = {0, P - 1} | (_last_tiles(1, P, 128, 1, False) if gemm else _last_tiles(OH, OW, BW, BH, up2))
    for p in pitches:
        pix |= _crossing_rows(p, P)
    g = torch.Generator().manual_seed(seed)
    pix |= set(torch.randint(0, P, (min(n_random, P),), generator=g).tolist())
    return torch.tensor(sorted(pix), dtype=torch.long)


def _attention_rows(T, n=256, seed=0):
    """About n query rows: four of the first 64-row block, all of the last (tail) query block, the last row, random."""
    last = (T - 1) // 64 * 64
    rows = {0, 1, 31, min(63, T - 1), T - 1} | set(range(last, T))
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, T, (max(n - len(rows), 0),), generator=g).tolist())
    return torch.tensor(sorted(rows), dtype=torch.long)


# ------------------------------------------------------------------------------------------------ float64 at samples
def _conv_ref_at(x, w, k, stride, pad, OW, cout, pix):
    """(sum a w, sum |a w|) float64 [len(pix), cout] of the convolution at flat output pixels pix (N = 1): the k x k x
    Cin patch of each gathered from x (zero outside), w [k*k, >= cout, Cin]."""
    _, H, W, Cin = x.shape
    pix = pix.to(x.device)
    oy, ox = pix // OW, pix % OW
    t = torch.arange(k * k, device=x.device)
    iy = oy[:, None] * stride + (t // k)[None] - pad[0]
    ix = ox[:, None] * stride + (t % k)[None] - pad[1]
    ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
    a = x[0, iy.clamp(0, H - 1), ix.clamp(0, W - 1), :Cin].double() * ok[..., None]
    wd = w[:, :cout, :Cin].double()
    return torch.einsum("ptc,toc->po", a, wd), torch.einsum("ptc,toc->po", a.abs(), wd.abs())


def _upconv_ref_at(x, w16, OW, cout, pix):
    """Nearest-2x upsample + 3x3 conv at output pixels pix: the four parity 2x2 convolutions over the folded taps, as
    test_gpu_vae_kernels._upconv64."""
    _, H, W, Cin = x.shape
    pix = pix.to(x.device)
    Y, X = pix // OW, pix % OW
    ref = torch.empty((len(pix), cout), dtype=torch.float64, device=x.device)
    mag = torch.empty_like(ref)
    for py in range(2):
        for px in range(2):
            sel = ((Y % 2) == py) & ((X % 2) == px)
            if not sel.any():
                continue
            i, j = Y[sel] // 2, X[sel] // 2
            t = torch.arange(4, device=x.device)
            iy = i[:, None] + py + (t // 2)[None] - 1
            ix = j[:, None] + px + (t % 2)[None] - 1
            ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
            a = x[0, iy.clamp(0, H - 1), ix.clamp(0, W - 1), :Cin].double() * ok[..., None]
            wd = w16[(py * 2 + px) * 4:(py * 2 + px) * 4 + 4, :cout, :Cin].double()
            ref[sel] = torch.einsum("ptc,toc->po", a, wd)
            mag[sel] = torch.einsum("ptc,toc->po", a.abs(), wd.abs())
    return ref, mag


def _nhwc_moments(x, groups, sms):
    """Float64 moments of every group of x [1, H, W, C] for the gn_stats_nhwc bound: mean, M2, R = max |x - mean|,
    S = sum (x - k)^2 over the kernel's own shifts k, the count n, n_t and D (module docstring).  In chunks of pixels."""
    _, H, W, C = x.shape
    P, cpg = H * W, C // groups
    chunk = (1 << 25) // C                                   # 256 MiB per float64 temporary
    xv = x.view(P, C)
    ppi = 256 // (C // 8)
    grid = max(1, min(-(-P // ppi), sms * 4))
    G = grid * ppi
    shifts = xv[:min(G, P), ::4].double()                    # k of each thread slot and 4-channel half
    tot = torch.zeros(groups, dtype=torch.float64, device=x.device)
    for s in range(0, P, chunk):
        tot += xv[s:s + chunk].double().view(-1, groups, cpg).sum(dim=(0, 2))
    n = P * cpg
    mu = tot / n
    m2 = torch.zeros_like(mu)
    R = torch.zeros_like(mu)
    S = torch.zeros_like(mu)
    for s in range(0, P, chunk):
        xc = xv[s:s + chunk].double()
        d = xc.view(-1, groups, cpg) - mu[None, :, None]
        m2 += (d * d).sum(dim=(0, 2))
        R = torch.maximum(R, d.abs().amax(dim=(0, 2)))
        k = shifts[torch.arange(s, s + xc.shape[0], device=x.device) % G].repeat_interleave(4, dim=1)
        sh = (xc - k).view(-1, groups, cpg)
        S += (sh * sh).sum(dim=(0, 2))
    n_t = 4 * -(-P // G)
    D = ppi * cpg // 4 + -(-grid // 32) + 5
    return dict(mu=mu, m2=m2, R=R, S=S, n=n, n_t=n_t, D=D)


def _check_nhwc_stats(var, mean, mom, dt, what):
    v64, e_mean, e_var = _stats_bounds(mom["mu"], mom["m2"], mom["R"], mom["S"], mom["n"], mom["n_t"], mom["D"], False,
                                       merge_roundings=(4, 6))
    assert torch.isfinite(mean).all() and torch.isfinite(var).all(), f"{what}: non-finite statistics"
    assert (var >= 0).all(), f"{what}: negative variance"
    em, ev = (mean.double() - mom["mu"]).abs(), (var.double() - v64).abs()
    rm, rv = (em / e_mean).max().item(), (ev / e_var).max().item()
    assert rm <= 1 and rv <= 1, f"{what}: mean err/bound {rm:.3g}, var err/bound {rv:.3g} (n = {mom['n']})"
    # the tolerances of test_gpu_vae_kernels._gn_stats_check as well: at these counts the worst-case bound allows
    # several times the variance itself (its n_t term grows with the per-thread count)
    tm, tv = (em / (2e-5 * mom["mu"].abs() + 2e-6)).max().item(), (ev / (5e-5 * v64 + 1e-6)).max().item()
    assert tm <= 1 and tv <= 1, f"{what}: mean err/tol {tm:.3g}, var err/tol {tv:.3g} (n = {mom['n']})"
    return max(rm, rv)


# ------------------------------------------------------------------------------------------------ one signature
def _peak_bytes(sig):
    """Device bytes one signature's replay holds at once, from its shapes (inputs, outputs, float64 work), + 2 GiB."""
    kind, e = sig[0], 2
    if kind == "conv":
        _, N, H, W, Cin, xp, cout, rows, k, stride, pt, pl, oh, ow, rp, act, dual, yp, bpr = sig
        b = N * H * W * xp + oh * ow * (yp + (cout if dual else 0) + rp)
    elif kind == "up2":
        _, N, H, W, Cin, cout, act, dual = sig
        b = H * W * Cin + 4 * H * W * cout * (2 if dual else 1)
    elif kind == "gemm":
        _, M, K, ap, n, brows, bp, yp, *_ = sig
        b = M * ap + brows * bp + M * yp
    elif kind == "attn":
        _, T, C, *_ = sig
        return 4 * T * C * e + 8 * 256 * T * 8 + 2 * GIB
    elif kind == "softmax":
        _, rows, pitch, cols, _ip = sig
        b = 2 * rows * pitch
    elif kind in ("gn_stats", "gn_apply"):
        _, H, W, C = sig[:4]
        b = 2 * H * W * C + GIB
    else:
        _, N, H, W, C = sig
        b = 5 * N * H * W * C
    return b * e + 2 * GIB


def _check_rows(got_rows, cols, v, bound, family, dt, what):
    """All `cols` values of each sampled pixel row within the bound; the row's pitch padding still NaN."""
    _within(got_rows[:, :cols], v, bound, family, dt, what)
    if got_rows.shape[1] > cols:
        assert torch.isnan(got_rows[:, cols:].float()).all(), f"{what}: pitch padding overwritten at a sampled pixel"


def _replay_large(sig, dt, seed):
    ops = _ops()
    kind = sig[0]
    what = f"{sig!r} {dt}"
    _need(_peak_bytes(sig), what)
    _reset()
    if kind == "conv":
        _, N, H, W, Cin, xp, cout, rows, k, stride, pt, pl, oh, ow, rp, act, dual, yp, bpr = sig
        assert N == 1 and rows == cout and not bpr
        x = _fill((1, H, W, xp), seed, dt, 0.7)[..., :Cin]
        w = _fill((k * k, cout, Cin), seed + 1, dt, (Cin * k * k) ** -0.5)
        bias = _fill((cout,), seed + 2, torch.float32, 0.3)
        rbuf = _fill((1, oh, ow, rp), seed + 3, dt, 0.5) if rp else None
        res = rbuf[..., :cout] if rp else None
        pst = None if act < 0 else (_fill((cout,), seed + 4, torch.float32, 0.4, 1.0), _fill((cout,), seed + 5, torch.float32, 0.2), bool(act))
        buf = _pitched_buf(oh * ow, cout, yp, dt)
        out = buf[:oh * ow].view(1, oh, ow, yp)[..., :cout]
        got = ops.conv2d_nhwc(x, w, bias, ksize=k, stride=stride, pad=(pt, pl), out_hw=(oh, ow), residual=res, out=out, post=pst, dual=dual)
        pix = _sample_pixels(oh, ow, [yp] + ([cout] if dual else []) + ([rp] if rp else []), seed=seed)
        ref, mag = _conv_ref_at(x, w, k, stride, (pt, pl), ow, cout, pix)
        pc = pix.cuda()
        v, e = _pre(ref, mag, k * k * Cin, 1.0, bias.double(), rbuf.view(-1, rp)[pc, :cout] if rp else None)
        y2 = got[1] if dual else None
        if pst is None or dual:
            _check_rows(buf[pc], cout, v, _out_bound(v, e, dt), "conv", dt, what)
        if pst is not None:
            z, ez = _post64(v, e, pst[0], pst[1], pst[2])
            rows_ = y2.reshape(-1, cout)[pc] if dual else buf[pc]
            _check_rows(rows_, cout, z, _out_bound(z, ez, dt), "conv+post", dt, what + (" (post)" if dual else ""))
        assert torch.isnan(buf[oh * ow:].float()).all(), f"{what}: wrote past the last pixel"
        del x, w, rbuf, res, buf, out, got, y2
    elif kind == "up2":
        _, N, H, W, Cin, cout, act, dual = sig
        x = _fill((1, H, W, Cin), seed, dt, 0.7)
        w16 = ops.fold_upsample_weight(_fill((cout, Cin, 3, 3), seed + 1, torch.float32, (Cin * 9) ** -0.5).to(dt), dt, cin_pad=Cin)
        bias = _fill((cout,), seed + 2, torch.float32, 0.3)
        pst = None if act < 0 else (_fill((cout,), seed + 4, torch.float32, 0.4, 1.0), _fill((cout,), seed + 5, torch.float32, 0.2), bool(act))
        got = ops.upconv2x_nhwc(x, w16, bias, post=pst, dual=dual)
        OH, OW = 2 * H, 2 * W
        pix = _sample_pixels(OH, OW, [cout], up2=True, seed=seed)
        ref, mag = _upconv_ref_at(x, w16, OW, cout, pix)
        pc = pix.cuda()
        v, e = _pre(ref, mag, 4 * Cin, 1.0, bias.double())
        y = got[0] if dual else got
        if pst is None or dual:
            _check_rows(y.reshape(-1, cout)[pc], cout, v, _out_bound(v, e, dt), "up2", dt, what)
        if pst is not None:
            z, ez = _post64(v, e, pst[0], pst[1], pst[2])
            _check_rows((got[1] if dual else got).reshape(-1, cout)[pc], cout, z, _out_bound(z, ez, dt), "up2+post", dt, what)
        del x, w16, got, y
    elif kind == "gemm":
        _, M, K, ap, n, brows, bp, yp, alpha, has_bias, bpr = sig
        a = _fill((M, ap), seed, dt, 0.5)
        a[:, K:] = 0
        b = _fill((brows, bp), seed + 1, dt, K ** -0.5)
        b[:, K:] = 0
        bv = _fill((M if bpr else n,), seed + 2, torch.float32, 0.3) if has_bias else None
        buf = _pitched_buf(M, n, yp, dt)
        ops.gemm_nt(a[:, :K], b[:, :K], bias=bv, alpha=alpha, n=n, out=buf[:M, :n], bias_per_row=bpr)
        rows = _sample_pixels(1, M, [yp, ap], gemm=True, seed=seed).cuda()
        ad, bd = a[rows, :K].double(), b[:n, :K].double()
        bb = None if bv is None else (bv.double()[rows][:, None] if bpr else bv.double()[None, :])
        v, e = _pre(ad @ bd.t(), ad.abs() @ bd.abs().t(), K, alpha, bb)
        _check_rows(buf[rows], n, v, _out_bound(v, e, dt), "gemm", dt, what)
        assert torch.isnan(buf[M:].float()).all(), f"{what}: wrote past the last row"
        del a, b, buf
    elif kind == "attn":
        _, T, C, *_r, alpha = sig
        q, k, v = (_fill((T, C), seed + i, dt, s, sh) for i, (s, sh) in enumerate([(1.7, 0.0), (1.7, 0.2), (1.0, 0.0)]))
        got = ops.attention(q, k, v, alpha)
        rows = _attention_rows(T, seed=seed).cuda()
        ref, bound = _attention64(q, k, v, alpha, dt, qidx=rows)
        _within(got[rows], ref, bound, "attention", dt, what)
        del q, k, v, got
    elif kind == "softmax":
        _, rows, pitch, cols, inplace = sig
        x = _fill((rows, pitch), seed, dt, 3.0)
        r = torch.tensor(sorted(_crossing_rows(pitch, rows) | {0, rows - 1} | set(range(0, rows, max(1, rows // 64)))), device="cuda")
        xr = x[r]
        y = ops.softmax_rows(x.clone(), cols) if inplace else ops.softmax_rows(x, cols)
        ref, bound = _softmax64(xr, cols, dt)
        _within(y[r, :cols], ref, bound, "softmax", dt, what)
        assert not y[r, cols:].any()
        if inplace:
            ops.softmax_rows(x, cols, out=x)
            assert torch.equal(x, y), f"{what}: in place differs from out of place"
        del x, y
    elif kind == "gn_stats":
        _, H, W, C, groups = sig
        x = _fill((1, H, W, C), seed, dt, 1.3, 0.8)
        var, mean = ops.gn_stats_nhwc(x, groups)
        _check_nhwc_stats(var, mean, _nhwc_moments(x, groups, torch.cuda.get_device_properties(0).multi_processor_count), dt, what)
        del x
    elif kind == "gn_apply":
        _, H, W, C, has_g, has_b, act = sig
        x = _fill((1, H, W, C), seed, dt, 1.3, 0.8)
        mean = _fill((32,), seed + 1, torch.float32, 0.3, 0.8)
        var = _fill((32,), seed + 2, torch.float32, 0.2).abs() + 0.5
        gamma = _fill((C,), seed + 3, torch.float32, 0.5, 1.0) if has_g else None
        beta = _fill((C,), seed + 4, torch.float32, 0.2) if has_b else None
        got = ops.gn_apply_nhwc(x, mean, var, gamma, beta, act)
        xv, gv = x.view(-1, C), got.view(-1, C)
        step = (1 << 24) // C
        for s in range(0, xv.shape[0], step):
            ref, bound = _gn_apply64(xv[s:s + step], mean, var, gamma, beta, act, dt)
            _within(gv[s:s + step], ref, bound, "gn_apply", dt, f"{what} pixels from {s}")
        del x, got
    elif kind == "up_nn":
        _, N, H, W, C = sig
        x = _fill((N, H, W, C), seed, dt)
        _upsample_bit_exact(x, ops.upsample2x_nhwc(x), what)
        del x
    else:
        raise AssertionError(f"unknown census entry {sig!r}")
    _track()


def _upsample_bit_exact(x, y, what, rows=64):
    for r0 in range(0, x.shape[1], rows):
        want = x[:, r0:r0 + rows].repeat_interleave(2, 1).repeat_interleave(2, 2)
        assert torch.equal(y[:, 2 * r0:2 * r0 + want.shape[1]].view(torch.int16), want.view(torch.int16)), f"{what}: rows from {r0}"


# ------------------------------------------------------------------------------------------------ 1. large census
# (is_decoder, H, W, tile[, one_tile]): one padded tile at the reference's 80 GB defaults (decoder 256, encoder 3072)
# and UI maxima (decoder 512, encoder 4096) -- VAEHook runs an input that small untiled, so it goes through
# vae_tile_forward, and it is exactly the interior tile of any larger input -- and one rectangular multi-tile input per
# direction, whose edge tiles are not square
LARGE_CENSUS_RUNS = [(True, 278, 278, 256, True), (True, 534, 534, 512, True), (False, 3136, 3136, 3072, True),
                     (False, 4160, 4160, 4096, True), (True, 320, 700, 256), (False, 3400, 4000, 3072)]

# recorded by record_census(LARGE_CENSUS_RUNS) on an H100 80GB HBM3: fp16 and bf16 (the same signatures), fast and slow mode
LARGE_CENSUS = [
    ('attn', 125184, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 147456, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 153664, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 262144, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 270400, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 285156, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 50596, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 53676, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 54528, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 55440, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 56320, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 65536, 512, 512, 512, 512, 0.04419417382415922),
    ('attn', 77284, 512, 512, 512, 512, 0.04419417382415922),
    ('conv', 1, 1024, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 1024, 1024, 0, -1, False, 256, False),
    ('conv', 1, 1024, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 1024, 1024, 256, -1, False, 256, False),
    ('conv', 1, 1024, 1024, 256, 256, 512, 512, 1, 1, 0, 0, 1024, 1024, 0, -1, False, 512, False),
    ('conv', 1, 1024, 1024, 256, 256, 512, 512, 3, 1, 1, 1, 1024, 1024, 0, -1, False, 512, False),
    ('conv', 1, 1024, 1024, 512, 512, 256, 256, 1, 1, 0, 0, 1024, 1024, 0, -1, False, 256, False),
    ('conv', 1, 1024, 1024, 512, 512, 256, 256, 3, 1, 1, 1, 1024, 1024, 0, -1, False, 256, False),
    ('conv', 1, 1024, 1024, 512, 512, 512, 512, 3, 1, 1, 1, 1024, 1024, 0, -1, False, 512, False),
    ('conv', 1, 1024, 1024, 512, 512, 512, 512, 3, 1, 1, 1, 1024, 1024, 512, -1, False, 512, False),
    ('conv', 1, 1024, 1024, 512, 512, 512, 512, 3, 2, 0, 0, 512, 512, 0, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 256, 256, 512, 512, 1, 1, 0, 0, 1040, 1040, 0, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 256, 256, 512, 512, 3, 1, 1, 1, 1040, 1040, 0, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 256, 256, 512, 512, 3, 1, 1, 1, 1040, 1040, 0, 1, False, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 1, 1, 1, 1040, 1040, 0, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 1, 1, 1, 1040, 1040, 0, 1, False, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 1, 1, 1, 1040, 1040, 512, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 1, 1, 1, 1040, 1040, 512, 1, True, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 2, 0, 0, 520, 520, 0, -1, False, 512, False),
    ('conv', 1, 1040, 1040, 512, 512, 512, 512, 3, 2, 0, 0, 520, 520, 0, 1, True, 512, False),
    ('conv', 1, 1068, 1068, 512, 512, 512, 512, 3, 1, 1, 1, 1068, 1068, 0, -1, False, 512, False),
    ('conv', 1, 1068, 1068, 512, 512, 512, 512, 3, 1, 1, 1, 1068, 1068, 0, 1, False, 512, False),
    ('conv', 1, 1068, 1068, 512, 512, 512, 512, 3, 1, 1, 1, 1068, 1068, 512, -1, False, 512, False),
    ('conv', 1, 1068, 1068, 512, 512, 512, 512, 3, 1, 1, 1, 1068, 1068, 512, 1, True, 512, False),
    ('conv', 1, 1112, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 1112, 1112, 0, -1, False, 256, False),
    ('conv', 1, 1112, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 1112, 1112, 0, 1, False, 256, False),
    ('conv', 1, 1112, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 1112, 1112, 256, -1, False, 256, False),
    ('conv', 1, 1112, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 1112, 1112, 256, 1, True, 256, False),
    ('conv', 1, 1112, 1112, 512, 512, 256, 256, 1, 1, 0, 0, 1112, 1112, 0, -1, False, 256, False),
    ('conv', 1, 1112, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 1112, 1112, 0, -1, False, 256, False),
    ('conv', 1, 1112, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 1112, 1112, 0, 1, False, 256, False),
    ('conv', 1, 117, 256, 512, 512, 512, 512, 1, 1, 0, 0, 117, 256, 512, -1, False, 512, False),
    ('conv', 1, 117, 256, 512, 512, 512, 512, 3, 1, 1, 1, 117, 256, 0, -1, False, 512, False),
    ('conv', 1, 117, 256, 512, 512, 512, 512, 3, 1, 1, 1, 117, 256, 512, -1, False, 512, False),
    ('conv', 1, 117, 256, 64, 64, 512, 512, 3, 1, 1, 1, 117, 256, 0, -1, False, 512, False),
    ('conv', 1, 1280, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1280, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 1504, 0, 1, False, 128, False),
    ('conv', 1, 1280, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 1504, 128, -1, False, 128, False),
    ('conv', 1, 1280, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 1504, 128, 1, False, 128, False),
    ('conv', 1, 1280, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 1504, 128, 1, True, 128, False),
    ('conv', 1, 1280, 1504, 128, 128, 16, 16, 3, 1, 1, 1, 1280, 1504, 0, -1, False, 16, False),
    ('conv', 1, 1280, 1504, 256, 256, 128, 128, 1, 1, 0, 0, 1280, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1280, 1504, 256, 256, 128, 128, 3, 1, 1, 1, 1280, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1280, 1504, 256, 256, 128, 128, 3, 1, 1, 1, 1280, 1504, 0, 1, False, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 2224, 0, 1, False, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 2224, 128, -1, False, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 2224, 128, 1, False, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1280, 2224, 128, 1, True, 128, False),
    ('conv', 1, 1280, 2224, 128, 128, 16, 16, 3, 1, 1, 1, 1280, 2224, 0, -1, False, 16, False),
    ('conv', 1, 1280, 2224, 256, 256, 128, 128, 1, 1, 0, 0, 1280, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1280, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 1280, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1280, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 1280, 2224, 0, 1, False, 128, False),
    ('conv', 1, 1305, 1536, 128, 128, 256, 256, 1, 1, 0, 0, 1305, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1305, 1536, 128, 128, 256, 256, 3, 1, 1, 1, 1305, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1305, 1536, 256, 256, 256, 256, 3, 1, 1, 1, 1305, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1305, 1536, 256, 256, 256, 256, 3, 1, 1, 1, 1305, 1536, 256, -1, False, 256, False),
    ('conv', 1, 1305, 1536, 256, 256, 256, 256, 3, 2, 0, 0, 652, 768, 0, -1, False, 256, False),
    ('conv', 1, 1456, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1456, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 1504, 0, 1, False, 128, False),
    ('conv', 1, 1456, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 1504, 128, -1, False, 128, False),
    ('conv', 1, 1456, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 1504, 128, 1, False, 128, False),
    ('conv', 1, 1456, 1504, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 1504, 128, 1, True, 128, False),
    ('conv', 1, 1456, 1504, 128, 128, 16, 16, 3, 1, 1, 1, 1456, 1504, 0, -1, False, 16, False),
    ('conv', 1, 1456, 1504, 256, 256, 128, 128, 1, 1, 0, 0, 1456, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1456, 1504, 256, 256, 128, 128, 3, 1, 1, 1, 1456, 1504, 0, -1, False, 128, False),
    ('conv', 1, 1456, 1504, 256, 256, 128, 128, 3, 1, 1, 1, 1456, 1504, 0, 1, False, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 2224, 0, 1, False, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 2224, 128, -1, False, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 2224, 128, 1, False, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 1456, 2224, 128, 1, True, 128, False),
    ('conv', 1, 1456, 2224, 128, 128, 16, 16, 3, 1, 1, 1, 1456, 2224, 0, -1, False, 16, False),
    ('conv', 1, 1456, 2224, 256, 256, 128, 128, 1, 1, 0, 0, 1456, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1456, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 1456, 2224, 0, -1, False, 128, False),
    ('conv', 1, 1456, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 1456, 2224, 0, 1, False, 128, False),
    ('conv', 1, 1536, 1536, 128, 128, 256, 256, 1, 1, 0, 0, 1536, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1536, 1536, 128, 128, 256, 256, 3, 1, 1, 1, 1536, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1536, 1536, 256, 256, 256, 256, 3, 1, 1, 1, 1536, 1536, 0, -1, False, 256, False),
    ('conv', 1, 1536, 1536, 256, 256, 256, 256, 3, 1, 1, 1, 1536, 1536, 256, -1, False, 256, False),
    ('conv', 1, 1536, 1536, 256, 256, 256, 256, 3, 2, 0, 0, 768, 768, 0, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 128, 128, 256, 256, 1, 1, 0, 0, 1568, 1568, 0, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 128, 128, 256, 256, 3, 1, 1, 1, 1568, 1568, 0, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 128, 128, 256, 256, 3, 1, 1, 1, 1568, 1568, 0, 1, False, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 1, 1, 1, 1568, 1568, 0, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 1, 1, 1, 1568, 1568, 0, 1, False, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 1, 1, 1, 1568, 1568, 256, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 1, 1, 1, 1568, 1568, 256, 1, True, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 2, 0, 0, 784, 784, 0, -1, False, 256, False),
    ('conv', 1, 1568, 1568, 256, 256, 256, 256, 3, 2, 0, 0, 784, 784, 0, 1, True, 256, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 1, 1, 0, 0, 160, 188, 512, -1, False, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 1, 1, 0, 0, 160, 188, 512, 1, True, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 3, 1, 1, 1, 160, 188, 0, -1, False, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 3, 1, 1, 1, 160, 188, 0, 1, False, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 3, 1, 1, 1, 160, 188, 512, -1, False, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 3, 1, 1, 1, 160, 188, 512, 0, True, 512, False),
    ('conv', 1, 160, 188, 512, 512, 512, 512, 3, 1, 1, 1, 160, 188, 512, 1, True, 512, False),
    ('conv', 1, 160, 188, 64, 64, 512, 512, 3, 1, 1, 1, 160, 188, 0, -1, False, 512, False),
    ('conv', 1, 160, 188, 64, 64, 512, 512, 3, 1, 1, 1, 160, 188, 0, 1, True, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 1, 1, 0, 0, 160, 278, 512, -1, False, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 1, 1, 0, 0, 160, 278, 512, 1, True, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 3, 1, 1, 1, 160, 278, 0, -1, False, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 3, 1, 1, 1, 160, 278, 0, 1, False, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 3, 1, 1, 1, 160, 278, 512, -1, False, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 3, 1, 1, 1, 160, 278, 512, 0, True, 512, False),
    ('conv', 1, 160, 278, 512, 512, 512, 512, 3, 1, 1, 1, 160, 278, 512, 1, True, 512, False),
    ('conv', 1, 160, 278, 64, 64, 512, 512, 3, 1, 1, 1, 160, 278, 0, -1, False, 512, False),
    ('conv', 1, 160, 278, 64, 64, 512, 512, 3, 1, 1, 1, 160, 278, 0, 1, True, 512, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2016, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2016, 0, 1, False, 128, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2016, 128, -1, False, 128, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2016, 128, 1, True, 128, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 2, 0, 0, 852, 1008, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2016, 128, 128, 128, 128, 3, 2, 0, 0, 852, 1008, 0, 1, True, 128, False),
    ('conv', 1, 1704, 2016, 64, 64, 128, 128, 3, 1, 1, 1, 1704, 2016, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2016, 64, 64, 128, 128, 3, 1, 1, 1, 1704, 2016, 0, 1, True, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2048, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2048, 0, 1, False, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2048, 128, -1, False, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1704, 2048, 128, 1, True, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 2, 0, 0, 852, 1024, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2048, 128, 128, 128, 128, 3, 2, 0, 0, 852, 1024, 0, 1, True, 128, False),
    ('conv', 1, 1704, 2048, 64, 64, 128, 128, 3, 1, 1, 1, 1704, 2048, 0, -1, False, 128, False),
    ('conv', 1, 1704, 2048, 64, 64, 128, 128, 3, 1, 1, 1, 1704, 2048, 0, 1, True, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2016, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2016, 0, 1, False, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2016, 128, -1, False, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2016, 128, 1, True, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 2, 0, 0, 880, 1008, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2016, 128, 128, 128, 128, 3, 2, 0, 0, 880, 1008, 0, 1, True, 128, False),
    ('conv', 1, 1760, 2016, 64, 64, 128, 128, 3, 1, 1, 1, 1760, 2016, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2016, 64, 64, 128, 128, 3, 1, 1, 1, 1760, 2016, 0, 1, True, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2048, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2048, 0, 1, False, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2048, 128, -1, False, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 1760, 2048, 128, 1, True, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 2, 0, 0, 880, 1024, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2048, 128, 128, 128, 128, 3, 2, 0, 0, 880, 1024, 0, 1, True, 128, False),
    ('conv', 1, 1760, 2048, 64, 64, 128, 128, 3, 1, 1, 1, 1760, 2048, 0, -1, False, 128, False),
    ('conv', 1, 1760, 2048, 64, 64, 128, 128, 3, 1, 1, 1, 1760, 2048, 0, 1, True, 128, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 1, 1, 0, 0, 182, 188, 512, -1, False, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 1, 1, 0, 0, 182, 188, 512, 1, True, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 3, 1, 1, 1, 182, 188, 0, -1, False, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 3, 1, 1, 1, 182, 188, 0, 1, False, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 3, 1, 1, 1, 182, 188, 512, -1, False, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 3, 1, 1, 1, 182, 188, 512, 0, True, 512, False),
    ('conv', 1, 182, 188, 512, 512, 512, 512, 3, 1, 1, 1, 182, 188, 512, 1, True, 512, False),
    ('conv', 1, 182, 188, 64, 64, 512, 512, 3, 1, 1, 1, 182, 188, 0, -1, False, 512, False),
    ('conv', 1, 182, 188, 64, 64, 512, 512, 3, 1, 1, 1, 182, 188, 0, 1, True, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 1, 1, 0, 0, 182, 278, 512, -1, False, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 1, 1, 0, 0, 182, 278, 512, 1, True, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 3, 1, 1, 1, 182, 278, 0, -1, False, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 3, 1, 1, 1, 182, 278, 0, 1, False, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 3, 1, 1, 1, 182, 278, 512, -1, False, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 3, 1, 1, 1, 182, 278, 512, 0, True, 512, False),
    ('conv', 1, 182, 278, 512, 512, 512, 512, 3, 1, 1, 1, 182, 278, 512, 1, True, 512, False),
    ('conv', 1, 182, 278, 64, 64, 512, 512, 3, 1, 1, 1, 182, 278, 0, -1, False, 512, False),
    ('conv', 1, 182, 278, 64, 64, 512, 512, 3, 1, 1, 1, 182, 278, 0, 1, True, 512, False),
    ('conv', 1, 2048, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 2048, 2048, 0, -1, False, 128, False),
    ('conv', 1, 2048, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 2048, 2048, 128, -1, False, 128, False),
    ('conv', 1, 2048, 2048, 128, 128, 256, 256, 1, 1, 0, 0, 2048, 2048, 0, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 128, 128, 256, 256, 3, 1, 1, 1, 2048, 2048, 0, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 256, 256, 128, 128, 1, 1, 0, 0, 2048, 2048, 0, -1, False, 128, False),
    ('conv', 1, 2048, 2048, 256, 256, 128, 128, 3, 1, 1, 1, 2048, 2048, 0, -1, False, 128, False),
    ('conv', 1, 2048, 2048, 256, 256, 256, 256, 3, 1, 1, 1, 2048, 2048, 0, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 256, 256, 256, 256, 3, 1, 1, 1, 2048, 2048, 256, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 256, 256, 256, 256, 3, 2, 0, 0, 1024, 1024, 0, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 512, 512, 256, 256, 1, 1, 0, 0, 2048, 2048, 0, -1, False, 256, False),
    ('conv', 1, 2048, 2048, 512, 512, 256, 256, 3, 1, 1, 1, 2048, 2048, 0, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 128, 128, 256, 256, 1, 1, 0, 0, 2080, 2080, 0, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 128, 128, 256, 256, 3, 1, 1, 1, 2080, 2080, 0, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 128, 128, 256, 256, 3, 1, 1, 1, 2080, 2080, 0, 1, False, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 1, 1, 1, 2080, 2080, 0, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 1, 1, 1, 2080, 2080, 0, 1, False, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 1, 1, 1, 2080, 2080, 256, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 1, 1, 1, 2080, 2080, 256, 1, True, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 2, 0, 0, 1040, 1040, 0, -1, False, 256, False),
    ('conv', 1, 2080, 2080, 256, 256, 256, 256, 3, 2, 0, 0, 1040, 1040, 0, 1, True, 256, False),
    ('conv', 1, 213, 252, 512, 512, 16, 16, 3, 1, 1, 1, 213, 252, 0, -1, False, 16, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 1, 1, 0, 0, 213, 252, 512, -1, False, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 1, 1, 0, 0, 213, 252, 512, 1, True, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 0, -1, False, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 0, 1, False, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 512, -1, False, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 512, 0, True, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 512, 1, False, 512, False),
    ('conv', 1, 213, 252, 512, 512, 512, 512, 3, 1, 1, 1, 213, 252, 512, 1, True, 512, False),
    ('conv', 1, 213, 256, 512, 512, 16, 16, 3, 1, 1, 1, 213, 256, 0, -1, False, 16, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 1, 1, 0, 0, 213, 256, 512, -1, False, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 1, 1, 0, 0, 213, 256, 512, 1, True, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 0, -1, False, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 0, 1, False, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 512, -1, False, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 512, 0, True, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 512, 1, False, 512, False),
    ('conv', 1, 213, 256, 512, 512, 512, 512, 3, 1, 1, 1, 213, 256, 512, 1, True, 512, False),
    ('conv', 1, 2136, 2136, 256, 256, 256, 256, 3, 1, 1, 1, 2136, 2136, 0, -1, False, 256, False),
    ('conv', 1, 2136, 2136, 256, 256, 256, 256, 3, 1, 1, 1, 2136, 2136, 0, 1, False, 256, False),
    ('conv', 1, 2136, 2136, 256, 256, 256, 256, 3, 1, 1, 1, 2136, 2136, 256, -1, False, 256, False),
    ('conv', 1, 2136, 2136, 256, 256, 256, 256, 3, 1, 1, 1, 2136, 2136, 256, 1, True, 256, False),
    ('conv', 1, 2136, 2136, 512, 512, 256, 256, 1, 1, 0, 0, 2136, 2136, 0, -1, False, 256, False),
    ('conv', 1, 2136, 2136, 512, 512, 256, 256, 3, 1, 1, 1, 2136, 2136, 0, -1, False, 256, False),
    ('conv', 1, 2136, 2136, 512, 512, 256, 256, 3, 1, 1, 1, 2136, 2136, 0, 1, False, 256, False),
    ('conv', 1, 220, 252, 512, 512, 16, 16, 3, 1, 1, 1, 220, 252, 0, -1, False, 16, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 1, 1, 0, 0, 220, 252, 512, -1, False, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 1, 1, 0, 0, 220, 252, 512, 1, True, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 0, -1, False, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 0, 1, False, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 512, -1, False, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 512, 0, True, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 512, 1, False, 512, False),
    ('conv', 1, 220, 252, 512, 512, 512, 512, 3, 1, 1, 1, 220, 252, 512, 1, True, 512, False),
    ('conv', 1, 220, 256, 512, 512, 16, 16, 3, 1, 1, 1, 220, 256, 0, -1, False, 16, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 1, 1, 0, 0, 220, 256, 512, -1, False, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 1, 1, 0, 0, 220, 256, 512, 1, True, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 0, -1, False, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 0, 1, False, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 512, -1, False, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 512, 0, True, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 512, 1, False, 512, False),
    ('conv', 1, 220, 256, 512, 512, 512, 512, 3, 1, 1, 1, 220, 256, 512, 1, True, 512, False),
    ('conv', 1, 2224, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 2224, 2224, 0, -1, False, 128, False),
    ('conv', 1, 2224, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 2224, 2224, 0, 1, False, 128, False),
    ('conv', 1, 2224, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 2224, 2224, 128, -1, False, 128, False),
    ('conv', 1, 2224, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 2224, 2224, 128, 1, False, 128, False),
    ('conv', 1, 2224, 2224, 128, 128, 128, 128, 3, 1, 1, 1, 2224, 2224, 128, 1, True, 128, False),
    ('conv', 1, 2224, 2224, 128, 128, 16, 16, 3, 1, 1, 1, 2224, 2224, 0, -1, False, 16, False),
    ('conv', 1, 2224, 2224, 256, 256, 128, 128, 1, 1, 0, 0, 2224, 2224, 0, -1, False, 128, False),
    ('conv', 1, 2224, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 2224, 2224, 0, -1, False, 128, False),
    ('conv', 1, 2224, 2224, 256, 256, 128, 128, 3, 1, 1, 1, 2224, 2224, 0, 1, False, 128, False),
    ('conv', 1, 234, 512, 512, 512, 512, 512, 3, 1, 1, 1, 234, 512, 0, -1, False, 512, False),
    ('conv', 1, 234, 512, 512, 512, 512, 512, 3, 1, 1, 1, 234, 512, 512, -1, False, 512, False),
    ('conv', 1, 256, 256, 512, 512, 512, 512, 1, 1, 0, 0, 256, 256, 512, -1, False, 512, False),
    ('conv', 1, 256, 256, 512, 512, 512, 512, 3, 1, 1, 1, 256, 256, 0, -1, False, 512, False),
    ('conv', 1, 256, 256, 512, 512, 512, 512, 3, 1, 1, 1, 256, 256, 512, -1, False, 512, False),
    ('conv', 1, 256, 256, 64, 64, 512, 512, 3, 1, 1, 1, 256, 256, 0, -1, False, 512, False),
    ('conv', 1, 2611, 3072, 128, 128, 128, 128, 3, 1, 1, 1, 2611, 3072, 0, -1, False, 128, False),
    ('conv', 1, 2611, 3072, 128, 128, 128, 128, 3, 1, 1, 1, 2611, 3072, 128, -1, False, 128, False),
    ('conv', 1, 2611, 3072, 128, 128, 128, 128, 3, 2, 0, 0, 1305, 1536, 0, -1, False, 128, False),
    ('conv', 1, 2611, 3072, 64, 64, 128, 128, 3, 1, 1, 1, 2611, 3072, 0, -1, False, 128, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 1, 1, 0, 0, 278, 278, 512, -1, False, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 1, 1, 0, 0, 278, 278, 512, 1, True, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 3, 1, 1, 1, 278, 278, 0, -1, False, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 3, 1, 1, 1, 278, 278, 0, 1, False, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 3, 1, 1, 1, 278, 278, 512, -1, False, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 3, 1, 1, 1, 278, 278, 512, 0, True, 512, False),
    ('conv', 1, 278, 278, 512, 512, 512, 512, 3, 1, 1, 1, 278, 278, 512, 1, True, 512, False),
    ('conv', 1, 278, 278, 64, 64, 512, 512, 3, 1, 1, 1, 278, 278, 0, -1, False, 512, False),
    ('conv', 1, 278, 278, 64, 64, 512, 512, 3, 1, 1, 1, 278, 278, 0, 1, True, 512, False),
    ('conv', 1, 3072, 3072, 128, 128, 128, 128, 3, 1, 1, 1, 3072, 3072, 0, -1, False, 128, False),
    ('conv', 1, 3072, 3072, 128, 128, 128, 128, 3, 1, 1, 1, 3072, 3072, 128, -1, False, 128, False),
    ('conv', 1, 3072, 3072, 128, 128, 128, 128, 3, 2, 0, 0, 1536, 1536, 0, -1, False, 128, False),
    ('conv', 1, 3072, 3072, 64, 64, 128, 128, 3, 1, 1, 1, 3072, 3072, 0, -1, False, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 1, 1, 1, 3136, 3136, 0, -1, False, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 1, 1, 1, 3136, 3136, 0, 1, False, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 1, 1, 1, 3136, 3136, 128, -1, False, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 1, 1, 1, 3136, 3136, 128, 1, True, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 2, 0, 0, 1568, 1568, 0, -1, False, 128, False),
    ('conv', 1, 3136, 3136, 128, 128, 128, 128, 3, 2, 0, 0, 1568, 1568, 0, 1, True, 128, False),
    ('conv', 1, 3136, 3136, 64, 64, 128, 128, 3, 1, 1, 1, 3136, 3136, 0, -1, False, 128, False),
    ('conv', 1, 3136, 3136, 64, 64, 128, 128, 3, 1, 1, 1, 3136, 3136, 0, 1, True, 128, False),
    ('conv', 1, 320, 376, 512, 512, 512, 512, 3, 1, 1, 1, 320, 376, 0, -1, False, 512, False),
    ('conv', 1, 320, 376, 512, 512, 512, 512, 3, 1, 1, 1, 320, 376, 0, 1, False, 512, False),
    ('conv', 1, 320, 376, 512, 512, 512, 512, 3, 1, 1, 1, 320, 376, 512, -1, False, 512, False),
    ('conv', 1, 320, 376, 512, 512, 512, 512, 3, 1, 1, 1, 320, 376, 512, 1, True, 512, False),
    ('conv', 1, 320, 556, 512, 512, 512, 512, 3, 1, 1, 1, 320, 556, 0, -1, False, 512, False),
    ('conv', 1, 320, 556, 512, 512, 512, 512, 3, 1, 1, 1, 320, 556, 0, 1, False, 512, False),
    ('conv', 1, 320, 556, 512, 512, 512, 512, 3, 1, 1, 1, 320, 556, 512, -1, False, 512, False),
    ('conv', 1, 320, 556, 512, 512, 512, 512, 3, 1, 1, 1, 320, 556, 512, 1, True, 512, False),
    ('conv', 1, 326, 384, 512, 512, 512, 512, 1, 1, 0, 0, 326, 384, 512, -1, False, 512, False),
    ('conv', 1, 326, 384, 512, 512, 512, 512, 3, 1, 1, 1, 326, 384, 0, -1, False, 512, False),
    ('conv', 1, 326, 384, 512, 512, 512, 512, 3, 1, 1, 1, 326, 384, 512, -1, False, 512, False),
    ('conv', 1, 364, 376, 512, 512, 512, 512, 3, 1, 1, 1, 364, 376, 0, -1, False, 512, False),
    ('conv', 1, 364, 376, 512, 512, 512, 512, 3, 1, 1, 1, 364, 376, 0, 1, False, 512, False),
    ('conv', 1, 364, 376, 512, 512, 512, 512, 3, 1, 1, 1, 364, 376, 512, -1, False, 512, False),
    ('conv', 1, 364, 376, 512, 512, 512, 512, 3, 1, 1, 1, 364, 376, 512, 1, True, 512, False),
    ('conv', 1, 364, 556, 512, 512, 512, 512, 3, 1, 1, 1, 364, 556, 0, -1, False, 512, False),
    ('conv', 1, 364, 556, 512, 512, 512, 512, 3, 1, 1, 1, 364, 556, 0, 1, False, 512, False),
    ('conv', 1, 364, 556, 512, 512, 512, 512, 3, 1, 1, 1, 364, 556, 512, -1, False, 512, False),
    ('conv', 1, 364, 556, 512, 512, 512, 512, 3, 1, 1, 1, 364, 556, 512, 1, True, 512, False),
    ('conv', 1, 384, 384, 512, 512, 512, 512, 1, 1, 0, 0, 384, 384, 512, -1, False, 512, False),
    ('conv', 1, 384, 384, 512, 512, 512, 512, 3, 1, 1, 1, 384, 384, 0, -1, False, 512, False),
    ('conv', 1, 384, 384, 512, 512, 512, 512, 3, 1, 1, 1, 384, 384, 512, -1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 16, 16, 3, 1, 1, 1, 392, 392, 0, -1, False, 16, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 1, 1, 0, 0, 392, 392, 512, -1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 1, 1, 0, 0, 392, 392, 512, 1, True, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 0, -1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 0, 1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 512, -1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 512, 0, True, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 512, 1, False, 512, False),
    ('conv', 1, 392, 392, 512, 512, 512, 512, 3, 1, 1, 1, 392, 392, 512, 1, True, 512, False),
    ('conv', 1, 4096, 4096, 128, 128, 128, 128, 3, 1, 1, 1, 4096, 4096, 0, -1, False, 128, False),
    ('conv', 1, 4096, 4096, 128, 128, 128, 128, 3, 1, 1, 1, 4096, 4096, 128, -1, False, 128, False),
    ('conv', 1, 4096, 4096, 128, 128, 128, 128, 3, 2, 0, 0, 2048, 2048, 0, -1, False, 128, False),
    ('conv', 1, 4096, 4096, 256, 256, 128, 128, 1, 1, 0, 0, 4096, 4096, 0, -1, False, 128, False),
    ('conv', 1, 4096, 4096, 256, 256, 128, 128, 3, 1, 1, 1, 4096, 4096, 0, -1, False, 128, False),
    ('conv', 1, 4096, 4096, 64, 64, 128, 128, 3, 1, 1, 1, 4096, 4096, 0, -1, False, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 1, 1, 1, 4160, 4160, 0, -1, False, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 1, 1, 1, 4160, 4160, 0, 1, False, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 1, 1, 1, 4160, 4160, 128, -1, False, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 1, 1, 1, 4160, 4160, 128, 1, True, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 2, 0, 0, 2080, 2080, 0, -1, False, 128, False),
    ('conv', 1, 4160, 4160, 128, 128, 128, 128, 3, 2, 0, 0, 2080, 2080, 0, 1, True, 128, False),
    ('conv', 1, 4160, 4160, 64, 64, 128, 128, 3, 1, 1, 1, 4160, 4160, 0, -1, False, 128, False),
    ('conv', 1, 4160, 4160, 64, 64, 128, 128, 3, 1, 1, 1, 4160, 4160, 0, 1, True, 128, False),
    ('conv', 1, 426, 504, 256, 256, 512, 512, 1, 1, 0, 0, 426, 504, 0, -1, False, 512, False),
    ('conv', 1, 426, 504, 256, 256, 512, 512, 3, 1, 1, 1, 426, 504, 0, -1, False, 512, False),
    ('conv', 1, 426, 504, 256, 256, 512, 512, 3, 1, 1, 1, 426, 504, 0, 1, False, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 1, 1, 1, 426, 504, 0, -1, False, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 1, 1, 1, 426, 504, 0, 1, False, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 1, 1, 1, 426, 504, 512, -1, False, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 1, 1, 1, 426, 504, 512, 1, True, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 2, 0, 0, 213, 252, 0, -1, False, 512, False),
    ('conv', 1, 426, 504, 512, 512, 512, 512, 3, 2, 0, 0, 213, 252, 0, 1, True, 512, False),
    ('conv', 1, 426, 512, 256, 256, 512, 512, 1, 1, 0, 0, 426, 512, 0, -1, False, 512, False),
    ('conv', 1, 426, 512, 256, 256, 512, 512, 3, 1, 1, 1, 426, 512, 0, -1, False, 512, False),
    ('conv', 1, 426, 512, 256, 256, 512, 512, 3, 1, 1, 1, 426, 512, 0, 1, False, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 1, 1, 1, 426, 512, 0, -1, False, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 1, 1, 1, 426, 512, 0, 1, False, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 1, 1, 1, 426, 512, 512, -1, False, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 1, 1, 1, 426, 512, 512, 1, True, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 2, 0, 0, 213, 256, 0, -1, False, 512, False),
    ('conv', 1, 426, 512, 512, 512, 512, 512, 3, 2, 0, 0, 213, 256, 0, 1, True, 512, False),
    ('conv', 1, 4272, 4272, 128, 128, 128, 128, 3, 1, 1, 1, 4272, 4272, 0, -1, False, 128, False),
    ('conv', 1, 4272, 4272, 128, 128, 128, 128, 3, 1, 1, 1, 4272, 4272, 0, 1, False, 128, False),
    ('conv', 1, 4272, 4272, 128, 128, 128, 128, 3, 1, 1, 1, 4272, 4272, 128, -1, False, 128, False),
    ('conv', 1, 4272, 4272, 128, 128, 128, 128, 3, 1, 1, 1, 4272, 4272, 128, 1, False, 128, False),
    ('conv', 1, 4272, 4272, 128, 128, 128, 128, 3, 1, 1, 1, 4272, 4272, 128, 1, True, 128, False),
    ('conv', 1, 4272, 4272, 128, 128, 16, 16, 3, 1, 1, 1, 4272, 4272, 0, -1, False, 16, False),
    ('conv', 1, 4272, 4272, 256, 256, 128, 128, 1, 1, 0, 0, 4272, 4272, 0, -1, False, 128, False),
    ('conv', 1, 4272, 4272, 256, 256, 128, 128, 3, 1, 1, 1, 4272, 4272, 0, -1, False, 128, False),
    ('conv', 1, 4272, 4272, 256, 256, 128, 128, 3, 1, 1, 1, 4272, 4272, 0, 1, False, 128, False),
    ('conv', 1, 440, 504, 256, 256, 512, 512, 1, 1, 0, 0, 440, 504, 0, -1, False, 512, False),
    ('conv', 1, 440, 504, 256, 256, 512, 512, 3, 1, 1, 1, 440, 504, 0, -1, False, 512, False),
    ('conv', 1, 440, 504, 256, 256, 512, 512, 3, 1, 1, 1, 440, 504, 0, 1, False, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 1, 1, 1, 440, 504, 0, -1, False, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 1, 1, 1, 440, 504, 0, 1, False, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 1, 1, 1, 440, 504, 512, -1, False, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 1, 1, 1, 440, 504, 512, 1, True, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 2, 0, 0, 220, 252, 0, -1, False, 512, False),
    ('conv', 1, 440, 504, 512, 512, 512, 512, 3, 2, 0, 0, 220, 252, 0, 1, True, 512, False),
    ('conv', 1, 440, 512, 256, 256, 512, 512, 1, 1, 0, 0, 440, 512, 0, -1, False, 512, False),
    ('conv', 1, 440, 512, 256, 256, 512, 512, 3, 1, 1, 1, 440, 512, 0, -1, False, 512, False),
    ('conv', 1, 440, 512, 256, 256, 512, 512, 3, 1, 1, 1, 440, 512, 0, 1, False, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 1, 1, 1, 440, 512, 0, -1, False, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 1, 1, 1, 440, 512, 0, 1, False, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 1, 1, 1, 440, 512, 512, -1, False, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 1, 1, 1, 440, 512, 512, 1, True, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 2, 0, 0, 220, 256, 0, -1, False, 512, False),
    ('conv', 1, 440, 512, 512, 512, 512, 512, 3, 2, 0, 0, 220, 256, 0, 1, True, 512, False),
    ('conv', 1, 468, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 468, 1024, 0, -1, False, 256, False),
    ('conv', 1, 468, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 468, 1024, 256, -1, False, 256, False),
    ('conv', 1, 468, 1024, 512, 512, 256, 256, 1, 1, 0, 0, 468, 1024, 0, -1, False, 256, False),
    ('conv', 1, 468, 1024, 512, 512, 256, 256, 3, 1, 1, 1, 468, 1024, 0, -1, False, 256, False),
    ('conv', 1, 512, 512, 512, 512, 512, 512, 1, 1, 0, 0, 512, 512, 512, -1, False, 512, False),
    ('conv', 1, 512, 512, 512, 512, 512, 512, 3, 1, 1, 1, 512, 512, 0, -1, False, 512, False),
    ('conv', 1, 512, 512, 512, 512, 512, 512, 3, 1, 1, 1, 512, 512, 512, -1, False, 512, False),
    ('conv', 1, 512, 512, 64, 64, 512, 512, 3, 1, 1, 1, 512, 512, 0, -1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 16, 16, 3, 1, 1, 1, 520, 520, 0, -1, False, 16, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 1, 1, 0, 0, 520, 520, 512, -1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 1, 1, 0, 0, 520, 520, 512, 1, True, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 0, -1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 0, 1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 512, -1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 512, 0, True, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 512, 1, False, 512, False),
    ('conv', 1, 520, 520, 512, 512, 512, 512, 3, 1, 1, 1, 520, 520, 512, 1, True, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 1, 1, 0, 0, 534, 534, 512, -1, False, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 1, 1, 0, 0, 534, 534, 512, 1, True, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 3, 1, 1, 1, 534, 534, 0, -1, False, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 3, 1, 1, 1, 534, 534, 0, 1, False, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 3, 1, 1, 1, 534, 534, 512, -1, False, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 3, 1, 1, 1, 534, 534, 512, 0, True, 512, False),
    ('conv', 1, 534, 534, 512, 512, 512, 512, 3, 1, 1, 1, 534, 534, 512, 1, True, 512, False),
    ('conv', 1, 534, 534, 64, 64, 512, 512, 3, 1, 1, 1, 534, 534, 0, -1, False, 512, False),
    ('conv', 1, 534, 534, 64, 64, 512, 512, 3, 1, 1, 1, 534, 534, 0, 1, True, 512, False),
    ('conv', 1, 556, 556, 512, 512, 512, 512, 3, 1, 1, 1, 556, 556, 0, -1, False, 512, False),
    ('conv', 1, 556, 556, 512, 512, 512, 512, 3, 1, 1, 1, 556, 556, 0, 1, False, 512, False),
    ('conv', 1, 556, 556, 512, 512, 512, 512, 3, 1, 1, 1, 556, 556, 512, -1, False, 512, False),
    ('conv', 1, 556, 556, 512, 512, 512, 512, 3, 1, 1, 1, 556, 556, 512, 1, True, 512, False),
    ('conv', 1, 640, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 640, 1112, 0, -1, False, 256, False),
    ('conv', 1, 640, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 640, 1112, 0, 1, False, 256, False),
    ('conv', 1, 640, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 640, 1112, 256, -1, False, 256, False),
    ('conv', 1, 640, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 640, 1112, 256, 1, True, 256, False),
    ('conv', 1, 640, 1112, 512, 512, 256, 256, 1, 1, 0, 0, 640, 1112, 0, -1, False, 256, False),
    ('conv', 1, 640, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 640, 1112, 0, -1, False, 256, False),
    ('conv', 1, 640, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 640, 1112, 0, 1, False, 256, False),
    ('conv', 1, 640, 752, 256, 256, 256, 256, 3, 1, 1, 1, 640, 752, 0, -1, False, 256, False),
    ('conv', 1, 640, 752, 256, 256, 256, 256, 3, 1, 1, 1, 640, 752, 0, 1, False, 256, False),
    ('conv', 1, 640, 752, 256, 256, 256, 256, 3, 1, 1, 1, 640, 752, 256, -1, False, 256, False),
    ('conv', 1, 640, 752, 256, 256, 256, 256, 3, 1, 1, 1, 640, 752, 256, 1, True, 256, False),
    ('conv', 1, 640, 752, 512, 512, 256, 256, 1, 1, 0, 0, 640, 752, 0, -1, False, 256, False),
    ('conv', 1, 640, 752, 512, 512, 256, 256, 3, 1, 1, 1, 640, 752, 0, -1, False, 256, False),
    ('conv', 1, 640, 752, 512, 512, 256, 256, 3, 1, 1, 1, 640, 752, 0, 1, False, 256, False),
    ('conv', 1, 652, 768, 256, 256, 512, 512, 1, 1, 0, 0, 652, 768, 0, -1, False, 512, False),
    ('conv', 1, 652, 768, 256, 256, 512, 512, 3, 1, 1, 1, 652, 768, 0, -1, False, 512, False),
    ('conv', 1, 652, 768, 512, 512, 512, 512, 3, 1, 1, 1, 652, 768, 0, -1, False, 512, False),
    ('conv', 1, 652, 768, 512, 512, 512, 512, 3, 1, 1, 1, 652, 768, 512, -1, False, 512, False),
    ('conv', 1, 652, 768, 512, 512, 512, 512, 3, 2, 0, 0, 326, 384, 0, -1, False, 512, False),
    ('conv', 1, 728, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 728, 1112, 0, -1, False, 256, False),
    ('conv', 1, 728, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 728, 1112, 0, 1, False, 256, False),
    ('conv', 1, 728, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 728, 1112, 256, -1, False, 256, False),
    ('conv', 1, 728, 1112, 256, 256, 256, 256, 3, 1, 1, 1, 728, 1112, 256, 1, True, 256, False),
    ('conv', 1, 728, 1112, 512, 512, 256, 256, 1, 1, 0, 0, 728, 1112, 0, -1, False, 256, False),
    ('conv', 1, 728, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 728, 1112, 0, -1, False, 256, False),
    ('conv', 1, 728, 1112, 512, 512, 256, 256, 3, 1, 1, 1, 728, 1112, 0, 1, False, 256, False),
    ('conv', 1, 728, 752, 256, 256, 256, 256, 3, 1, 1, 1, 728, 752, 0, -1, False, 256, False),
    ('conv', 1, 728, 752, 256, 256, 256, 256, 3, 1, 1, 1, 728, 752, 0, 1, False, 256, False),
    ('conv', 1, 728, 752, 256, 256, 256, 256, 3, 1, 1, 1, 728, 752, 256, -1, False, 256, False),
    ('conv', 1, 728, 752, 256, 256, 256, 256, 3, 1, 1, 1, 728, 752, 256, 1, True, 256, False),
    ('conv', 1, 728, 752, 512, 512, 256, 256, 1, 1, 0, 0, 728, 752, 0, -1, False, 256, False),
    ('conv', 1, 728, 752, 512, 512, 256, 256, 3, 1, 1, 1, 728, 752, 0, -1, False, 256, False),
    ('conv', 1, 728, 752, 512, 512, 256, 256, 3, 1, 1, 1, 728, 752, 0, 1, False, 256, False),
    ('conv', 1, 768, 768, 256, 256, 512, 512, 1, 1, 0, 0, 768, 768, 0, -1, False, 512, False),
    ('conv', 1, 768, 768, 256, 256, 512, 512, 3, 1, 1, 1, 768, 768, 0, -1, False, 512, False),
    ('conv', 1, 768, 768, 512, 512, 512, 512, 3, 1, 1, 1, 768, 768, 0, -1, False, 512, False),
    ('conv', 1, 768, 768, 512, 512, 512, 512, 3, 1, 1, 1, 768, 768, 512, -1, False, 512, False),
    ('conv', 1, 768, 768, 512, 512, 512, 512, 3, 2, 0, 0, 384, 384, 0, -1, False, 512, False),
    ('conv', 1, 784, 784, 256, 256, 512, 512, 1, 1, 0, 0, 784, 784, 0, -1, False, 512, False),
    ('conv', 1, 784, 784, 256, 256, 512, 512, 3, 1, 1, 1, 784, 784, 0, -1, False, 512, False),
    ('conv', 1, 784, 784, 256, 256, 512, 512, 3, 1, 1, 1, 784, 784, 0, 1, False, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 1, 1, 1, 784, 784, 0, -1, False, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 1, 1, 1, 784, 784, 0, 1, False, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 1, 1, 1, 784, 784, 512, -1, False, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 1, 1, 1, 784, 784, 512, 1, True, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 2, 0, 0, 392, 392, 0, -1, False, 512, False),
    ('conv', 1, 784, 784, 512, 512, 512, 512, 3, 2, 0, 0, 392, 392, 0, 1, True, 512, False),
    ('conv', 1, 852, 1008, 128, 128, 256, 256, 1, 1, 0, 0, 852, 1008, 0, -1, False, 256, False),
    ('conv', 1, 852, 1008, 128, 128, 256, 256, 3, 1, 1, 1, 852, 1008, 0, -1, False, 256, False),
    ('conv', 1, 852, 1008, 128, 128, 256, 256, 3, 1, 1, 1, 852, 1008, 0, 1, False, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1008, 0, -1, False, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1008, 0, 1, False, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1008, 256, -1, False, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1008, 256, 1, True, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 2, 0, 0, 426, 504, 0, -1, False, 256, False),
    ('conv', 1, 852, 1008, 256, 256, 256, 256, 3, 2, 0, 0, 426, 504, 0, 1, True, 256, False),
    ('conv', 1, 852, 1024, 128, 128, 256, 256, 1, 1, 0, 0, 852, 1024, 0, -1, False, 256, False),
    ('conv', 1, 852, 1024, 128, 128, 256, 256, 3, 1, 1, 1, 852, 1024, 0, -1, False, 256, False),
    ('conv', 1, 852, 1024, 128, 128, 256, 256, 3, 1, 1, 1, 852, 1024, 0, 1, False, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1024, 0, -1, False, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1024, 0, 1, False, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1024, 256, -1, False, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 852, 1024, 256, 1, True, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 2, 0, 0, 426, 512, 0, -1, False, 256, False),
    ('conv', 1, 852, 1024, 256, 256, 256, 256, 3, 2, 0, 0, 426, 512, 0, 1, True, 256, False),
    ('conv', 1, 880, 1008, 128, 128, 256, 256, 1, 1, 0, 0, 880, 1008, 0, -1, False, 256, False),
    ('conv', 1, 880, 1008, 128, 128, 256, 256, 3, 1, 1, 1, 880, 1008, 0, -1, False, 256, False),
    ('conv', 1, 880, 1008, 128, 128, 256, 256, 3, 1, 1, 1, 880, 1008, 0, 1, False, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1008, 0, -1, False, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1008, 0, 1, False, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1008, 256, -1, False, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1008, 256, 1, True, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 2, 0, 0, 440, 504, 0, -1, False, 256, False),
    ('conv', 1, 880, 1008, 256, 256, 256, 256, 3, 2, 0, 0, 440, 504, 0, 1, True, 256, False),
    ('conv', 1, 880, 1024, 128, 128, 256, 256, 1, 1, 0, 0, 880, 1024, 0, -1, False, 256, False),
    ('conv', 1, 880, 1024, 128, 128, 256, 256, 3, 1, 1, 1, 880, 1024, 0, -1, False, 256, False),
    ('conv', 1, 880, 1024, 128, 128, 256, 256, 3, 1, 1, 1, 880, 1024, 0, 1, False, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1024, 0, -1, False, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1024, 0, 1, False, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1024, 256, -1, False, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 1, 1, 1, 880, 1024, 256, 1, True, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 2, 0, 0, 440, 512, 0, -1, False, 256, False),
    ('conv', 1, 880, 1024, 256, 256, 256, 256, 3, 2, 0, 0, 440, 512, 0, 1, True, 256, False),
    ('conv', 1, 936, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 936, 2048, 0, -1, False, 128, False),
    ('conv', 1, 936, 2048, 128, 128, 128, 128, 3, 1, 1, 1, 936, 2048, 128, -1, False, 128, False),
    ('conv', 1, 936, 2048, 256, 256, 128, 128, 1, 1, 0, 0, 936, 2048, 0, -1, False, 128, False),
    ('conv', 1, 936, 2048, 256, 256, 128, 128, 3, 1, 1, 1, 936, 2048, 0, -1, False, 128, False),
    ('gemm', 125184, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 147456, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 153664, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 262144, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 270400, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 285156, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 29952, 29952, 29952, 512, 512, 29952, 512, 1.0, False, False),
    ('gemm', 29952, 512, 512, 29952, 29952, 512, 29952, 0.04419417382415922, False, False),
    ('gemm', 29952, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 30080, 30080, 30080, 512, 512, 30080, 512, 1.0, False, False),
    ('gemm', 30080, 512, 512, 30080, 30080, 512, 30080, 0.04419417382415922, False, False),
    ('gemm', 30080, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 34216, 34216, 34216, 512, 512, 34216, 512, 1.0, False, False),
    ('gemm', 34216, 512, 512, 34216, 34216, 512, 34216, 0.04419417382415922, False, False),
    ('gemm', 34216, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 44480, 44480, 44480, 512, 512, 44480, 512, 1.0, False, False),
    ('gemm', 44480, 512, 512, 44480, 44480, 512, 44480, 0.04419417382415922, False, False),
    ('gemm', 44480, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 50596, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 512, 512, 512, 29952, 29952, 512, 29952, 1.0, True, True),
    ('gemm', 512, 512, 512, 30080, 30080, 512, 30080, 1.0, True, True),
    ('gemm', 512, 512, 512, 34216, 34216, 512, 34216, 1.0, True, True),
    ('gemm', 512, 512, 512, 44480, 44480, 512, 44480, 1.0, True, True),
    ('gemm', 53676, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 54528, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 55440, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 56320, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 65536, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gemm', 77284, 512, 512, 512, 512, 512, 512, 1.0, True, False),
    ('gn_apply', 1024, 1024, 256, True, True, True),
    ('gn_apply', 1024, 1024, 512, True, True, True),
    ('gn_apply', 1040, 1040, 256, True, True, True),
    ('gn_apply', 1040, 1040, 512, True, True, True),
    ('gn_apply', 1068, 1068, 512, True, True, True),
    ('gn_apply', 1112, 1112, 256, True, True, True),
    ('gn_apply', 1112, 1112, 512, True, True, True),
    ('gn_apply', 117, 256, 512, True, True, False),
    ('gn_apply', 117, 256, 512, True, True, True),
    ('gn_apply', 1280, 1504, 128, True, True, True),
    ('gn_apply', 1280, 1504, 256, True, True, True),
    ('gn_apply', 1280, 2224, 128, True, True, True),
    ('gn_apply', 1280, 2224, 256, True, True, True),
    ('gn_apply', 1305, 1536, 128, True, True, True),
    ('gn_apply', 1305, 1536, 256, True, True, True),
    ('gn_apply', 1456, 1504, 128, True, True, True),
    ('gn_apply', 1456, 1504, 256, True, True, True),
    ('gn_apply', 1456, 2224, 128, True, True, True),
    ('gn_apply', 1456, 2224, 256, True, True, True),
    ('gn_apply', 1536, 1536, 128, True, True, True),
    ('gn_apply', 1536, 1536, 256, True, True, True),
    ('gn_apply', 1568, 1568, 128, True, True, True),
    ('gn_apply', 1568, 1568, 256, True, True, True),
    ('gn_apply', 160, 188, 512, True, True, False),
    ('gn_apply', 160, 188, 512, True, True, True),
    ('gn_apply', 160, 278, 512, True, True, False),
    ('gn_apply', 160, 278, 512, True, True, True),
    ('gn_apply', 1704, 2016, 128, True, True, True),
    ('gn_apply', 1704, 2048, 128, True, True, True),
    ('gn_apply', 1760, 2016, 128, True, True, True),
    ('gn_apply', 1760, 2048, 128, True, True, True),
    ('gn_apply', 182, 188, 512, True, True, False),
    ('gn_apply', 182, 188, 512, True, True, True),
    ('gn_apply', 182, 278, 512, True, True, False),
    ('gn_apply', 182, 278, 512, True, True, True),
    ('gn_apply', 2048, 2048, 128, True, True, True),
    ('gn_apply', 2048, 2048, 256, True, True, True),
    ('gn_apply', 2048, 2048, 512, True, True, True),
    ('gn_apply', 2080, 2080, 128, True, True, True),
    ('gn_apply', 2080, 2080, 256, True, True, True),
    ('gn_apply', 213, 252, 512, True, True, False),
    ('gn_apply', 213, 252, 512, True, True, True),
    ('gn_apply', 213, 256, 512, True, True, False),
    ('gn_apply', 213, 256, 512, True, True, True),
    ('gn_apply', 2136, 2136, 256, True, True, True),
    ('gn_apply', 2136, 2136, 512, True, True, True),
    ('gn_apply', 220, 252, 512, True, True, False),
    ('gn_apply', 220, 252, 512, True, True, True),
    ('gn_apply', 220, 256, 512, True, True, False),
    ('gn_apply', 220, 256, 512, True, True, True),
    ('gn_apply', 2224, 2224, 128, True, True, True),
    ('gn_apply', 2224, 2224, 256, True, True, True),
    ('gn_apply', 234, 512, 512, True, True, True),
    ('gn_apply', 256, 256, 512, True, True, False),
    ('gn_apply', 256, 256, 512, True, True, True),
    ('gn_apply', 2611, 3072, 128, True, True, True),
    ('gn_apply', 278, 278, 512, True, True, False),
    ('gn_apply', 278, 278, 512, True, True, True),
    ('gn_apply', 3072, 3072, 128, True, True, True),
    ('gn_apply', 3136, 3136, 128, True, True, True),
    ('gn_apply', 320, 376, 512, True, True, True),
    ('gn_apply', 320, 556, 512, True, True, True),
    ('gn_apply', 326, 384, 512, True, True, False),
    ('gn_apply', 326, 384, 512, True, True, True),
    ('gn_apply', 364, 376, 512, True, True, True),
    ('gn_apply', 364, 556, 512, True, True, True),
    ('gn_apply', 384, 384, 512, True, True, False),
    ('gn_apply', 384, 384, 512, True, True, True),
    ('gn_apply', 392, 392, 512, True, True, False),
    ('gn_apply', 392, 392, 512, True, True, True),
    ('gn_apply', 4096, 4096, 128, True, True, True),
    ('gn_apply', 4096, 4096, 256, True, True, True),
    ('gn_apply', 4160, 4160, 128, True, True, True),
    ('gn_apply', 426, 504, 256, True, True, True),
    ('gn_apply', 426, 504, 512, True, True, True),
    ('gn_apply', 426, 512, 256, True, True, True),
    ('gn_apply', 426, 512, 512, True, True, True),
    ('gn_apply', 4272, 4272, 128, True, True, True),
    ('gn_apply', 4272, 4272, 256, True, True, True),
    ('gn_apply', 440, 504, 256, True, True, True),
    ('gn_apply', 440, 504, 512, True, True, True),
    ('gn_apply', 440, 512, 256, True, True, True),
    ('gn_apply', 440, 512, 512, True, True, True),
    ('gn_apply', 468, 1024, 256, True, True, True),
    ('gn_apply', 468, 1024, 512, True, True, True),
    ('gn_apply', 512, 512, 512, True, True, False),
    ('gn_apply', 512, 512, 512, True, True, True),
    ('gn_apply', 520, 520, 512, True, True, False),
    ('gn_apply', 520, 520, 512, True, True, True),
    ('gn_apply', 534, 534, 512, True, True, False),
    ('gn_apply', 534, 534, 512, True, True, True),
    ('gn_apply', 556, 556, 512, True, True, True),
    ('gn_apply', 640, 1112, 256, True, True, True),
    ('gn_apply', 640, 1112, 512, True, True, True),
    ('gn_apply', 640, 752, 256, True, True, True),
    ('gn_apply', 640, 752, 512, True, True, True),
    ('gn_apply', 652, 768, 256, True, True, True),
    ('gn_apply', 652, 768, 512, True, True, True),
    ('gn_apply', 728, 1112, 256, True, True, True),
    ('gn_apply', 728, 1112, 512, True, True, True),
    ('gn_apply', 728, 752, 256, True, True, True),
    ('gn_apply', 728, 752, 512, True, True, True),
    ('gn_apply', 768, 768, 256, True, True, True),
    ('gn_apply', 768, 768, 512, True, True, True),
    ('gn_apply', 784, 784, 256, True, True, True),
    ('gn_apply', 784, 784, 512, True, True, True),
    ('gn_apply', 852, 1008, 128, True, True, True),
    ('gn_apply', 852, 1008, 256, True, True, True),
    ('gn_apply', 852, 1024, 128, True, True, True),
    ('gn_apply', 852, 1024, 256, True, True, True),
    ('gn_apply', 880, 1008, 128, True, True, True),
    ('gn_apply', 880, 1008, 256, True, True, True),
    ('gn_apply', 880, 1024, 128, True, True, True),
    ('gn_apply', 880, 1024, 256, True, True, True),
    ('gn_apply', 936, 2048, 128, True, True, True),
    ('gn_apply', 936, 2048, 256, True, True, True),
    ('gn_stats', 1024, 1024, 256, 32),
    ('gn_stats', 1024, 1024, 512, 32),
    ('gn_stats', 1040, 1040, 256, 32),
    ('gn_stats', 1040, 1040, 512, 32),
    ('gn_stats', 1068, 1068, 512, 32),
    ('gn_stats', 1112, 1112, 256, 32),
    ('gn_stats', 1112, 1112, 512, 32),
    ('gn_stats', 117, 256, 512, 32),
    ('gn_stats', 1280, 1504, 128, 32),
    ('gn_stats', 1280, 1504, 256, 32),
    ('gn_stats', 1280, 2224, 128, 32),
    ('gn_stats', 1280, 2224, 256, 32),
    ('gn_stats', 1305, 1536, 128, 32),
    ('gn_stats', 1305, 1536, 256, 32),
    ('gn_stats', 1456, 1504, 128, 32),
    ('gn_stats', 1456, 1504, 256, 32),
    ('gn_stats', 1456, 2224, 128, 32),
    ('gn_stats', 1456, 2224, 256, 32),
    ('gn_stats', 1536, 1536, 128, 32),
    ('gn_stats', 1536, 1536, 256, 32),
    ('gn_stats', 1568, 1568, 128, 32),
    ('gn_stats', 1568, 1568, 256, 32),
    ('gn_stats', 160, 188, 512, 32),
    ('gn_stats', 160, 278, 512, 32),
    ('gn_stats', 1704, 2016, 128, 32),
    ('gn_stats', 1704, 2048, 128, 32),
    ('gn_stats', 1760, 2016, 128, 32),
    ('gn_stats', 1760, 2048, 128, 32),
    ('gn_stats', 182, 188, 512, 32),
    ('gn_stats', 182, 278, 512, 32),
    ('gn_stats', 2048, 2048, 128, 32),
    ('gn_stats', 2048, 2048, 256, 32),
    ('gn_stats', 2048, 2048, 512, 32),
    ('gn_stats', 2080, 2080, 128, 32),
    ('gn_stats', 2080, 2080, 256, 32),
    ('gn_stats', 213, 252, 512, 32),
    ('gn_stats', 213, 256, 512, 32),
    ('gn_stats', 2136, 2136, 256, 32),
    ('gn_stats', 2136, 2136, 512, 32),
    ('gn_stats', 220, 252, 512, 32),
    ('gn_stats', 220, 256, 512, 32),
    ('gn_stats', 2224, 2224, 128, 32),
    ('gn_stats', 2224, 2224, 256, 32),
    ('gn_stats', 234, 512, 512, 32),
    ('gn_stats', 256, 256, 512, 32),
    ('gn_stats', 2611, 3072, 128, 32),
    ('gn_stats', 278, 278, 512, 32),
    ('gn_stats', 3072, 3072, 128, 32),
    ('gn_stats', 3136, 3136, 128, 32),
    ('gn_stats', 320, 376, 512, 32),
    ('gn_stats', 320, 556, 512, 32),
    ('gn_stats', 326, 384, 512, 32),
    ('gn_stats', 364, 376, 512, 32),
    ('gn_stats', 364, 556, 512, 32),
    ('gn_stats', 384, 384, 512, 32),
    ('gn_stats', 392, 392, 512, 32),
    ('gn_stats', 4096, 4096, 128, 32),
    ('gn_stats', 4096, 4096, 256, 32),
    ('gn_stats', 4160, 4160, 128, 32),
    ('gn_stats', 426, 504, 256, 32),
    ('gn_stats', 426, 504, 512, 32),
    ('gn_stats', 426, 512, 256, 32),
    ('gn_stats', 426, 512, 512, 32),
    ('gn_stats', 4272, 4272, 128, 32),
    ('gn_stats', 4272, 4272, 256, 32),
    ('gn_stats', 440, 504, 256, 32),
    ('gn_stats', 440, 504, 512, 32),
    ('gn_stats', 440, 512, 256, 32),
    ('gn_stats', 440, 512, 512, 32),
    ('gn_stats', 468, 1024, 256, 32),
    ('gn_stats', 468, 1024, 512, 32),
    ('gn_stats', 512, 512, 512, 32),
    ('gn_stats', 520, 520, 512, 32),
    ('gn_stats', 534, 534, 512, 32),
    ('gn_stats', 556, 556, 512, 32),
    ('gn_stats', 640, 1112, 256, 32),
    ('gn_stats', 640, 1112, 512, 32),
    ('gn_stats', 640, 752, 256, 32),
    ('gn_stats', 640, 752, 512, 32),
    ('gn_stats', 652, 768, 256, 32),
    ('gn_stats', 652, 768, 512, 32),
    ('gn_stats', 728, 1112, 256, 32),
    ('gn_stats', 728, 1112, 512, 32),
    ('gn_stats', 728, 752, 256, 32),
    ('gn_stats', 728, 752, 512, 32),
    ('gn_stats', 768, 768, 256, 32),
    ('gn_stats', 768, 768, 512, 32),
    ('gn_stats', 784, 784, 256, 32),
    ('gn_stats', 784, 784, 512, 32),
    ('gn_stats', 852, 1008, 128, 32),
    ('gn_stats', 852, 1008, 256, 32),
    ('gn_stats', 852, 1024, 128, 32),
    ('gn_stats', 852, 1024, 256, 32),
    ('gn_stats', 880, 1008, 128, 32),
    ('gn_stats', 880, 1008, 256, 32),
    ('gn_stats', 880, 1024, 128, 32),
    ('gn_stats', 880, 1024, 256, 32),
    ('gn_stats', 936, 2048, 128, 32),
    ('gn_stats', 936, 2048, 256, 32),
    ('softmax', 29952, 29952, 29952, True),
    ('softmax', 30080, 30080, 30080, True),
    ('softmax', 34216, 34216, 34216, True),
    ('softmax', 44480, 44480, 44480, True),
    ('up2', 1, 1024, 1024, 256, 256, -1, False),
    ('up2', 1, 1024, 1024, 512, 512, -1, False),
    ('up2', 1, 1068, 1068, 512, 512, -1, False),
    ('up2', 1, 1068, 1068, 512, 512, 1, True),
    ('up2', 1, 1112, 1112, 256, 256, -1, False),
    ('up2', 1, 1112, 1112, 256, 256, 1, True),
    ('up2', 1, 117, 256, 512, 512, -1, False),
    ('up2', 1, 160, 188, 512, 512, -1, False),
    ('up2', 1, 160, 188, 512, 512, 1, True),
    ('up2', 1, 160, 278, 512, 512, -1, False),
    ('up2', 1, 160, 278, 512, 512, 1, True),
    ('up2', 1, 182, 188, 512, 512, -1, False),
    ('up2', 1, 182, 188, 512, 512, 1, True),
    ('up2', 1, 182, 278, 512, 512, -1, False),
    ('up2', 1, 182, 278, 512, 512, 1, True),
    ('up2', 1, 2048, 2048, 256, 256, -1, False),
    ('up2', 1, 2136, 2136, 256, 256, -1, False),
    ('up2', 1, 2136, 2136, 256, 256, 1, True),
    ('up2', 1, 234, 512, 512, 512, -1, False),
    ('up2', 1, 256, 256, 512, 512, -1, False),
    ('up2', 1, 278, 278, 512, 512, -1, False),
    ('up2', 1, 278, 278, 512, 512, 1, True),
    ('up2', 1, 320, 376, 512, 512, -1, False),
    ('up2', 1, 320, 376, 512, 512, 1, True),
    ('up2', 1, 320, 556, 512, 512, -1, False),
    ('up2', 1, 320, 556, 512, 512, 1, True),
    ('up2', 1, 364, 376, 512, 512, -1, False),
    ('up2', 1, 364, 376, 512, 512, 1, True),
    ('up2', 1, 364, 556, 512, 512, -1, False),
    ('up2', 1, 364, 556, 512, 512, 1, True),
    ('up2', 1, 468, 1024, 256, 256, -1, False),
    ('up2', 1, 512, 512, 512, 512, -1, False),
    ('up2', 1, 534, 534, 512, 512, -1, False),
    ('up2', 1, 534, 534, 512, 512, 1, True),
    ('up2', 1, 556, 556, 512, 512, -1, False),
    ('up2', 1, 556, 556, 512, 512, 1, True),
    ('up2', 1, 640, 1112, 256, 256, -1, False),
    ('up2', 1, 640, 1112, 256, 256, 1, True),
    ('up2', 1, 640, 752, 256, 256, -1, False),
    ('up2', 1, 640, 752, 256, 256, 1, True),
    ('up2', 1, 728, 1112, 256, 256, -1, False),
    ('up2', 1, 728, 1112, 256, 256, 1, True),
    ('up2', 1, 728, 752, 256, 256, -1, False),
    ('up2', 1, 728, 752, 256, 256, 1, True),
]


@pytest.mark.gpu
def test_large_census_is_complete():
    """Re-run the spy at the large tiles: every signature the engine issues there is in LARGE_CENSUS, and the census
    reaches the sizes this file exists for."""
    t0 = time.time()
    _reset()
    seen = record_census(LARGE_CENSUS_RUNS)
    _track()
    missing = [s for s in seen if s not in set(LARGE_CENSUS)]
    assert not missing, f"{len(missing)} signatures missing from LARGE_CENSUS, e.g. {missing[:5]}"
    print(f"large census: {len(seen)} signatures seen, {len(LARGE_CENSUS)} committed, {time.time() - t0:.1f} s")
    attn = {s[1] for s in LARGE_CENSUS if s[0] == "attn"}
    assert {77284, 153664, 270400, 285156} <= attn, sorted(attn)
    assert any(s[1] * s[2] * (s[3] // s[4]) > 2 ** 24 for s in LARGE_CENSUS if s[0] == "gn_stats"), "a GroupNorm group past 2^24 elements"


def _elements_out(sig):
    if sig[0] == "conv":
        return sig[12] * sig[13] * sig[17]
    if sig[0] == "up2":
        return 4 * sig[2] * sig[3] * sig[5]
    return 0


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_large_census_signatures_against_float64(dn):
    """Every LARGE_CENSUS signature on random data: dense kernels at the sampled pixels, the rest whole."""
    dt = DTS[dn]
    assert any(_elements_out(s) > 2 ** 31 for s in LARGE_CENSUS), "no output past 2^31 elements in the census"
    t0 = time.time()
    for i, sig in enumerate(LARGE_CENSUS):
        _replay_large(sig, dt, 5000 + 17 * i)
        torch.cuda.empty_cache()
    print(f"large census {dn}: {len(LARGE_CENSUS)} signatures in {time.time() - t0:.1f} s, peak {PEAK['bytes'] / 1e9:.1f} GB")


@pytest.mark.gpu
def test_sample_positions_hold_the_crossings():
    """For every dense LARGE_CENSUS output past 2^30 elements, the sample holds each crossing element's pixel and every
    pixel of the last pixel tiles (the checks above rely on it)."""
    seen = 0
    for sig in LARGE_CENSUS:
        if sig[0] not in ("conv", "up2") or _elements_out(sig) <= 2 ** 30:
            continue
        up2 = sig[0] == "up2"
        oh, ow, pitch = (2 * sig[2], 2 * sig[3], sig[5]) if up2 else (sig[12], sig[13], sig[17])
        pix = set(_sample_pixels(oh, ow, [pitch], up2=up2).tolist())
        for e in CROSSINGS:
            if e < oh * ow * pitch:
                assert {(e - 1) // pitch, e // pitch} <= pix, (sig, e)
                seen += 1
        assert _last_tiles(oh, ow, *_pixel_tile(oh, ow, up2), up2) <= pix
    assert seen >= 2


# ------------------------------------------------------------------------------------------------ 3. attention path boundary
def _attention_backend(dt, seed):
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    torch.manual_seed(seed)
    mod = types.SimpleNamespace(**{n: torch.nn.Conv2d(512, 512, 1).cuda().to(dt) for n in ("q", "k", "v", "proj_out")})
    return ve, ve.TensorCoreBackend(types.SimpleNamespace(cache={}), torch.device("cuda"), dt), types.SimpleNamespace(module=mod)


def _traced(ve, names, hook):
    """Wrap vae_engine.ops functions: hook(name, args, kwargs, call) runs instead of each and returns its result."""
    real = {n: getattr(ve.ops, n) for n in names}

    class Ctx:
        def __enter__(self):
            for n in names:
                setattr(ve.ops, n, (lambda n_: lambda *a, **kw: hook(n_, a, kw, real[n_]))(n))

        def __exit__(self, *exc):
            for n in names:
                setattr(ve.ops, n, real[n])
    return Ctx()


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_four_gemm_attention_at_the_largest_tile(dn):
    """T = SCORE_MATRIX_MAX_TOKENS = 46340 through TensorCoreBackend.attention: the four-GEMM path, whose [T, Tp] score
    matrix (Tp = 46344) holds 2^31 + 97312 elements.  The score GEMM rows around and past the 2^30 and 2^31 element
    crossings, softmax_rows there and P V at sampled rows against float64."""
    dt = DTS[dn]
    ve, be, op = _attention_backend(dt, 7)
    T, C = 46340, 512
    assert T == ve.SCORE_MATRIX_MAX_TOKENS
    Tp = _ops().round_up(T, 8)
    assert T * Tp > 2 ** 31
    _need(T * Tp * 2 + 10 * T * C * 2 + 4 * GIB, f"four-GEMM attention T={T}")
    _reset()
    rows = torch.tensor(sorted(_crossing_rows(Tp, T) | set(range(T - 4, T)) | set(_attention_rows(T, 64, 3).tolist())), device="cuda")
    assert max(rows.tolist()) * Tp >= 2 ** 31
    log = {}

    def hook(name, a, kw, call):
        if name == "softmax_rows":
            log["s_in"] = a[0][rows].clone()
            out = call(*a, **kw)
            log["s_out"] = out[rows].clone()
            return out
        if name == "gemm_nt":
            log.setdefault("gemm", []).append((a, kw))
        if name == "attention":
            log["fused"] = True
        out = call(*a, **kw)
        if name == "gemm_nt":
            log["gemm"][-1] += (out,)
        return out
    a = _fill((1, 140, 331, C), 11, dt, 0.7)
    with _traced(ve, ("gemm_nt", "softmax_rows", "attention"), hook):
        be.attention(a, op, None)
    assert "fused" not in log and "s_in" in log, "T = 46340 must take the four-GEMM path"
    alpha = float(int(C) ** -0.5)
    (q, k), skw, _ = log["gemm"][3][0], log["gemm"][3][1], None
    assert skw["alpha"] == alpha and log["gemm"][3][2].stride(0) == Tp
    qd, kd = q[rows].double(), k.double()
    v_, e_ = _pre(qd @ kd.t(), qd.abs() @ kd.abs().t(), C, alpha)
    _within(log["s_in"][:, :T], v_, _out_bound(v_, e_, dt), "gemm", dt, f"S rows T={T} {dn}")    # s is torch.empty: no sentinel
    del v_, e_
    ref, bound = _softmax64(log["s_in"], T, dt)
    _within(log["s_out"][:, :T], ref, bound, "softmax", dt, f"softmax rows T={T} {dn}")
    assert not log["s_out"][:, T:].any()
    (p, vt), _kw, o = log["gemm"][4]
    assert p.shape == (T, Tp) and vt.shape == (C, Tp)
    assert torch.equal(p[rows], log["s_out"])
    pd, vd = p[rows].double(), vt.double()
    v_, e_ = _pre(pd @ vd.t(), pd.abs() @ vd.abs().t(), Tp)
    _within(o[rows], v_, _out_bound(v_, e_, dt), "gemm", dt, f"P V rows T={T} {dn}")
    _track()


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_fused_attention_just_past_the_four_gemm_limit(dn):
    """T = 46341 through TensorCoreBackend.attention takes the fused kernel; 256 query rows against float64."""
    dt = DTS[dn]
    ve, be, op = _attention_backend(dt, 8)
    T, C = 46341, 512
    assert T == ve.SCORE_MATRIX_MAX_TOKENS + 1
    _need(10 * T * C * 2 + 2 * GIB, f"fused attention T={T}")
    log = {}

    def hook(name, a, kw, call):
        out = call(*a, **kw)
        log.setdefault(name, []).append((a, kw, out))
        return out
    with _traced(ve, ("softmax_rows", "attention"), hook):
        be.attention(_fill((1, 171, 271, C), 12, dt, 0.7), op, None)
    assert "softmax_rows" not in log and len(log.get("attention", [])) == 1, "T = 46341 must take the fused kernel"
    (q, k, v, alpha), _kw, out = log["attention"][0]
    rows = _attention_rows(T, seed=5).cuda()
    ref, bound = _attention64(q, k, v, alpha, dt, qidx=rows)
    _within(out[rows], ref, bound, "attention", dt, f"fused T={T} {dn}")
    _track()


# ------------------------------------------------------------------------------------------------ layout kernels, whole
@pytest.mark.gpu
@pytest.mark.parametrize("dn", DN)
def test_layout_kernels_past_2_31_bytes_bit_exact(dn):
    """nchw_to_nhwc and nchw_to_nhwc_wrap at the encoder-4096 tile load ([1, 3, 4160, 4160] -> [1, 4160, 4160, 64],
    2.2 GB), nhwc_to_nchw_region of a 128-channel [1, 4272, 4272] tile (2^31 + 1.9e8 elements each side) into a wider
    canvas, and upsample2x_nhwc to [1, 4272, 4272, 128]: bit-exact over the whole tensor, chunk by chunk."""
    dt = DTS[dn]
    ops = _ops()
    _need(4 * 4272 * 4272 * 128 * 2 + 2 * GIB, "layout kernels")
    _reset()
    z = _fill((1, 3, 4200, 4300), 20, dt)
    for bbox in [(17, 17 + 4160, 23, 23 + 4160), (-70, 4090, -41, 4119)]:
        y0, x0 = bbox[2], bbox[0]
        got = ops.nchw_to_nhwc(z[:, :, y0:y0 + 4160, x0:x0 + 4160], 64) if x0 >= 0 else ops.nchw_to_nhwc_wrap(z, bbox, 64)
        assert got.numel() * 2 > 2 ** 31
        for r0 in range(0, 4160, 256):
            ry = torch.arange(y0 + r0, y0 + min(r0 + 256, 4160), device="cuda") % 4200
            rx = torch.arange(x0, x0 + 4160, device="cuda") % 4300
            want = z[:, :, ry][:, :, :, rx].permute(0, 2, 3, 1)
            blk = got[:, r0:r0 + 256]
            assert torch.equal(blk[..., :3].view(torch.int16), want.view(torch.int16)), f"{bbox} rows from {r0}"
            assert not blk[..., 3:].view(torch.int16).any()
        del got
    del z
    x = _fill((1, 4272, 4272, 128), 21, dt)
    dst = torch.full((1, 128, 4272, 4280), 3.0, dtype=dt, device="cuda")
    ops.nhwc_to_nchw_region(x, dst[:, :, :, 5:5 + 4272], 128)
    for c0 in range(0, 128, 8):
        want = x[..., c0:c0 + 8].permute(0, 3, 1, 2)
        assert torch.equal(dst[:, c0:c0 + 8, :, 5:5 + 4272].view(torch.int16), want.view(torch.int16)), f"channels from {c0}"
        assert (dst[:, c0:c0 + 8, :, :5] == 3).all() and (dst[:, c0:c0 + 8, :, 5 + 4272:] == 3).all()
    del dst
    x = x[:, :2136, :2136].contiguous()
    _upsample_bit_exact(x, ops.upsample2x_nhwc(x), f"upsample2x {dn}")
    _track()


# ------------------------------------------------------------------------------------------------ 4. fp32 NCHW kernels
@pytest.mark.gpu
def test_fp32_module_backend_kernels_past_2_31_elements():
    """td_gn_stats, td_gn_apply and td_copy_region (the module backend's GroupNorm and tile copy) on an fp32
    [1, 512, 2136, 2136] activation (2.34e9 elements, 9.3 GB) against float64 in chunks, with the bounds of
    test_gpu_vae_nchw_kernels.py."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    dt, B, C, H, W, groups = torch.float32, 1, 512, 2136, 2136, 32
    _need(2 * C * H * (W + 8) * 4 + 6 * GIB, "fp32 NCHW kernels")
    _reset()
    x = _fill((B, C, H, W), 30, dt, 1.3, 0.8)
    assert x.numel() > 2 ** 31
    var, mean = tilevae.get_var_mean(x, groups)
    seg = C // groups * H * W
    chunk, chunks, _vec = plan_stats(groups, seg, 4)
    n_t = -(-chunk // (STAT_THREADS * 4)) * 4
    D = 13 + -(-chunks // 32)
    xs = x.view(groups, seg)
    for g in range(groups):
        s = xs[g].double()
        mu = s.mean()
        dev = s - mu
        m2, R = (dev * dev).sum(), dev.abs().max()
        del dev
        sh = s - s[::chunk].repeat_interleave(chunk)[:seg]
        S = (sh * sh).sum()
        del sh, s
        v64, e_mean, e_var = _stats_bounds(mu, m2, R, S, seg, n_t, D, False)
        rm, rv = ((mean[g].double() - mu).abs() / e_mean).item(), ((var[g].double() - v64).abs() / e_var).item()
        assert rm <= 1 and rv <= 1, f"group {g}: mean err/bound {rm:.3g}, var err/bound {rv:.3g}"
    gamma, beta = _fill((C,), 31, dt, 0.5, 1.0), _fill((C,), 32, dt, 0.3)
    y = tilevae.custom_group_norm(x, groups, mean, var, gamma, beta, act=True)
    cpg = C // groups
    for g in range(groups):
        sl = slice(g * cpg, (g + 1) * cpg)
        ref, bound = _apply64(x[:, sl].reshape(1, cpg, H * W), mean[g:g + 1], var[g:g + 1], gamma[sl], beta[sl], True, 1, False)
        _within_nchw(y[:, sl].reshape(1, cpg, H * W), ref, bound, "gn_apply", dt, f"fp32 group {g}")
        del ref, bound
    del y
    dst = torch.full((B, C, H, W + 8), 7.0, dtype=dt, device="cuda")
    tilevae.copy_region(x, dst[:, :, :, 3:3 + W])
    for c0 in range(0, C, 32):
        assert torch.equal(dst[:, c0:c0 + 32, :, 3:3 + W].view(torch.int32), x[:, c0:c0 + 32].view(torch.int32)), f"planes from {c0}"
        assert (dst[:, c0:c0 + 32, :, :3] == 7).all() and (dst[:, c0:c0 + 32, :, 3 + W:] == 7).all()
    _track()


# ------------------------------------------------------------------------------------------------ 5. UI maxima end to end
@pytest.mark.gpu
@pytest.mark.parametrize("is_dec,L,tile,T", [(True, 534, 512, 285156), (False, 4160, 4096, 270400)], ids=["decoder512", "encoder4096"])
def test_ui_maximum_tile_runs(is_dec, L, tile, T):
    """One padded tile at the UI's largest tile size, fp16, fast mode, through the wgmma backend: completes with the
    right shape and finite output, its mid-block attention runs T tokens, and every kernel call is in LARGE_CENSUS."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    from oracle import synth
    dt = torch.float16
    net = _sd_width_net(is_dec, 3 if is_dec else 4).cuda().to(dt)
    fp = ve.tile_footprint(ve.compile_program(net, is_dec), "wgmma", dt, L, L, 1)
    out_c = net.conv_out.out_channels
    oh = L * 8 if is_dec else L // 8
    _need(fp.working + out_c * oh * oh * 2 + 2 * GIB, f"{'decoder' if is_dec else 'encoder'} tile {tile}")
    _reset()
    z = synth.latent(5 if is_dec else 6, (1, 4 if is_dec else 3, L, L), dt).cuda()
    hook = tilevae.VAEHook(net, tile, is_dec, fast_decoder=True, fast_encoder=True, color_fix=False)
    t0 = time.time()
    with census_spy() as seen, torch.no_grad():
        out = hook.vae_tile_forward(z)
    torch.cuda.synchronize()
    print(f"{'decoder' if is_dec else 'encoder'} tile {tile}: {time.time() - t0:.1f} s, peak {(torch.cuda.max_memory_allocated() - PEAK['base']) / 1e9:.1f} GB")
    assert hook.backend_name == "wgmma"
    assert out.shape == (1, out_c, oh, oh) and torch.isfinite(out).all()
    assert T in {s[1] for s in seen if s[0] == "attn"}
    missing = [s for s in seen if s not in set(LARGE_CENSUS)]
    assert not missing, f"{len(missing)} calls not in LARGE_CENSUS, e.g. {missing[:3]}"
    _track()


@pytest.mark.gpu
def test_zz_report_peak_memory():
    print(f"peak device memory of this file (above what other tests hold): {PEAK['bytes'] / 1e9:.1f} GB")


# ------------------------------------------------------------------------------------------------ 6. the checkers fail (no GPU)
def _fails(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def test_sampled_checkers_catch_injected_defects():
    """Each sampled checker, fed the exact (rounded) result with one defect injected, fails; fed the exact result, it
    passes.  On the CPU, at the real decoder-512 level-0 shape: the input is a strided view of a small buffer (pixel
    (i, j) holds row i + j), so only the sampled patches are ever read."""
    dt, H, W, C = torch.float16, 4272, 4272, 128
    g = torch.Generator().manual_seed(1)
    base = (torch.randn((H + W, C), generator=g) * 0.7).to(dt)
    x = base.as_strided((1, H, W, C), (0, C, C, 1))
    w = (torch.randn((9, C, C), generator=g) * (9 * C) ** -0.5).to(dt)
    pix = _sample_pixels(H, W, [C], seed=2)
    ref, mag = _conv_ref_at(x, w, 3, 1, (1, 1), W, C, pix)
    v, e = _pre(ref, mag, 9 * C)
    bound = _out_bound(v, e, dt)
    good = v.to(dt)
    _check_rows(good, C, v, bound, "conv", dt, "exact")
    # one element wrong at the 2^31 crossing: it takes its neighbour channel's value (an index off by one there)
    r = int((pix == 2 ** 31 // C).nonzero())
    bad = good.clone()
    bad[r, 2 ** 31 % C] = good[r, 2 ** 31 % C + 1]
    assert _fails(lambda: _check_rows(bad, C, v, bound, "conv", dt, "crossing"))
    # the last pixel tile (the corner: 4272 = 534 x 8 = 267 x 16, so it is whole here) left unwritten (zeroed output)
    last = torch.tensor([i for i, p in enumerate(pix.tolist()) if p // W >= (H - 1) // 8 * 8 and p % W >= (W - 1) // 16 * 16])
    assert len(last) == (H - (H - 1) // 8 * 8) * (W - (W - 1) // 16 * 16)
    bad = good.clone()
    bad[last] = 0
    assert _fails(lambda: _check_rows(bad, C, v, bound, "conv", dt, "last tile"))
    # attention with the tail query block zeroed (T = 4100: a 4-row tail block, as T = 285156 has a 36-row one)
    T, Ca = 4100, 64
    q, k, vv = ((torch.randn((T, Ca), generator=g) * s).to(dt) for s in (1.7, 1.7, 1.0))
    rows = _attention_rows(T, seed=3)
    assert set(range(4096, T)) <= set(rows.tolist()) and T - 1 in rows.tolist()
    aref, abound = _attention64(q, k, vv, Ca ** -0.5, dt, qidx=rows)
    got = aref.to(dt)
    _within(got, aref, abound, "attention", dt, "exact")
    got[rows >= 4096] = 0
    assert _fails(lambda: _within(got, aref, abound, "attention", dt, "tail rows"))
    # gn_stats: a group of the decoder-512 level-0 activation (4 channels x 4272^2 pixels), as moments of N(0.8, 1.3^2)
    n = 4 * H * W
    assert n > 2 ** 24
    grid, ppi = 132 * 4, 16
    mom = dict(mu=torch.tensor([0.8], dtype=torch.float64), m2=torch.tensor([1.69 * n], dtype=torch.float64),
               R=torch.tensor([1.3 * 6.0], dtype=torch.float64), S=torch.tensor([2 * 1.69 * n], dtype=torch.float64), n=n,
               n_t=4 * -(-(H * W) // (grid * ppi)), D=ppi + -(-grid // 32) + 5)
    exact_var = (mom["m2"] / n).float()
    _check_nhwc_stats(exact_var, mom["mu"].float(), mom, dt, "exact")
    stalled = (mom["m2"] / 2 ** 24).float()           # a float counter that adds 1 stops at 2^24
    assert _fails(lambda: _check_nhwc_stats(stalled, mom["mu"].float(), mom, dt, "count stalled at 2^24"))
    assert float(torch.tensor(float(n), dtype=torch.float32)) == n
