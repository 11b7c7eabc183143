"""DemoFusion's device entry points at every scale the UI offers (1..8) and in every dtype, against plain references.

  td_dilated_gather             == torch.cat of the reference's strided slices            bit for bit
  td_demofusion_combine(_offset) == the reference's eager `+=` / `/ 2` / mix in the dtype  bit for bit
  td_depthwise_conv2d           vs float64 (and vs F.conv2d in the dtype on the GPU)       rounding bound
  td_gn_stats (nseg 1, unbiased) vs float64 mean / unbiased variance                       rtol of test_gpu_vae
  td_affine_clamp               == (g - m) / sd * so + mo evaluated eagerly in the dtype     bit for bit
  DemoFusion.sample_one_step    vs oracle.demofusion.sample_one_step                       tests/test_demofusion.py tolerances

The argument refusals run without a GPU: every bad argument is refused before any launch, so the pointers they pass
are never read.
"""
import ctypes
import math
import random
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import demofusion as odf
from oracle import synth, tiling
from oracle.make_golden import demo_denoise, position_aware_denoise

DTS = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
SCALES = list(range(1, 9))          # the UI's scale factor slider (scripts/tileglobal.py of the reference)
MAX_VIEWS = 64                      # kMaxViews of csrc/td_demofusion.cu: views per td_dilated_gather launch
MAX_KERNEL = 15                     # kMaxKernel: 2 * 8 - 1 taps


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def _stream():
    return _cabi().current_stream_ptr() if torch.cuda.is_available() else None


def _i32(v):
    return (ctypes.c_int32 * len(v))(*[int(i) for i in v])


def _with_outliers(x: torch.Tensor, seed: int, near_max: bool = True) -> torch.Tensor:
    """`x` with a few deliberate outliers in place: odd multiples of the smallest subnormal (where `acc * 0.5` has to
    round), values near the dtype's maximum (positive only, so overflow gives +inf and never inf - inf), signed zeros
    and the smallest normals of both signs."""
    fi = torch.finfo(x.dtype)
    tiny_sub = fi.tiny * fi.eps           # smallest subnormal
    big = [0.75 * fi.max, 0.6 * fi.max] if near_max else [3.0, -2.5]
    special = [3 * tiny_sub, -3 * tiny_sub, 5 * tiny_sub, -tiny_sub, *big, 0.0, -0.0, fi.tiny, -fi.tiny]
    flat = x.reshape(-1)
    rng = np.random.Generator(np.random.PCG64(seed))
    n = min(flat.numel(), 4 * len(special))
    idx = rng.choice(flat.numel(), size=n, replace=False)
    vals = torch.tensor([special[i % len(special)] for i in range(n)], dtype=torch.float64).to(x.dtype)
    flat[torch.from_numpy(idx)] = vals
    return x


def _latent(seed, shape, dt, outliers=True, near_max=True):
    x = synth.latent(seed, shape, dt)
    return _with_outliers(x, seed + 1, near_max) if outliers else x


def _views(s: int, mixture: bool):
    return odf.global_views(s, mixture)


# ------------------------------------------------------------------------------------------------ canvases
def _canvas(kind: str, s: int, off: int):
    """(H, W, end_y, end_x, oh, ow) of a canvas whose views satisfy the reference's equal-views rule: the slices
    `by + off:end:s` with `end = W - off` (both axes, demofusion.py:280) all have oh rows and ow columns.  Portrait
    canvases end their views at end_y = min(H, end) < H - off, so rows past it get x_global = 0."""
    ow = max(9, 40 // s)
    end_x = off + s * ow
    W = end_x + off
    if kind == "landscape":
        H = off + s * max(5, 28 // s)              # no bottom margin: end_y = H
    elif kind == "portrait":
        H = W + 2 * s + 3
    else:
        H = W
    end_y = min(H, end_x)
    assert (end_y - off) % s == 0 and (end_x - off) % s == 0
    return H, W, end_y, end_x, (end_y - off) // s, ow


CANVASES = ["landscape", "portrait", "square"]


# ------------------------------------------------------------------------------------------------ refusals (CPU)
def _scratch(nbytes=4096):
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    return torch.zeros(nbytes, dtype=torch.uint8, device=dev)


def _last_error():
    return _cabi().lib.td_last_error().decode()


def _combine_args(**over):
    """A valid td_demofusion_combine argument set (4x4 views at s = 2 on an 8x8 canvas, mixture off), with overrides."""
    buf = _scratch()
    a = dict(N=1, C=1, H=8, W=8, s=2, out_h=4, out_w=4, end_y=8, end_x=8, mixture=0, n_views=4, num_batches=1, vpb=4)
    a.update(over)
    ptrs = (ctypes.c_void_p * max(1, a["num_batches"]))(*([buf.data_ptr()] * max(1, a["num_batches"])))
    return buf, ptrs, a


def _call_combine(a, ptrs, buf, offset=None):
    lib = _cabi().lib
    common = (a["N"], a["C"], a["H"], a["W"], a["s"], a["out_h"], a["out_w"])
    tail = (a["end_y"], a["end_x"], a["mixture"], 0.25, 0.75, _cabi().TD_F16, _stream())
    out = buf.data_ptr() + buf.numel() // 2          # x_local and the views in the first half, out in the second
    if offset is None:
        return lib.td_demofusion_combine(buf.data_ptr(), ptrs, a["num_batches"], a["vpb"], a["n_views"], out, *common, *tail)
    return lib.td_demofusion_combine_offset(buf.data_ptr(), ptrs, a["num_batches"], a["vpb"], a["n_views"], out, *common, offset, *tail)


BAD_COMBINE = {
    "s0": dict(s=0, n_views=0),                       # passes n_views == s*s; the kernel would compute y % 0
    "s_negative": dict(s=-1, n_views=1),
    "N0": dict(N=0), "C0": dict(C=0), "H0": dict(H=0, end_y=0), "W0": dict(W=0, end_x=0),
    "out_h0": dict(out_h=0), "out_w0": dict(out_w=0),
    "end_y_past_H": dict(end_y=9), "end_x_past_W": dict(end_x=9),
    "rows_not_covered": dict(H=12, W=12, end_y=12),   # rows 8..11 would read past the 4-row views
    "cols_not_covered": dict(H=12, W=12, end_x=12),
    "rows_and_cols_not_covered": dict(H=12, W=12, end_y=12, end_x=12),
    "too_many_batches": dict(num_batches=129, vpb=1, s=8, n_views=64),
    "views_short": dict(num_batches=1, vpb=3),
}


@pytest.mark.parametrize("case", list(BAD_COMBINE), ids=list(BAD_COMBINE))
def test_combine_refuses_bad_arguments(case):
    """Every bad argument is refused with TD_ERR_INVALID_ARG and a message naming the call, by td_demofusion_combine and
    by its jitter sibling td_demofusion_combine_offset (offset 0) alike."""
    cabi = _cabi()
    buf, ptrs, a = _combine_args(**BAD_COMBINE[case])
    for offset, name in ((None, "td_demofusion_combine"), (0, "td_demofusion_combine_offset")):
        st = _call_combine(a, ptrs, buf, offset)
        msg = _last_error()
        assert st == cabi.TD_ERR_INVALID_ARG, f"{name} {case}: status {st} ({msg})"
        assert msg.startswith(name + ":"), msg
        if "covered" in case:
            assert "do not cover" in msg, msg


def test_combine_accepts_the_valid_base_arguments():
    """The refusals above differ from an accepted call only in the named argument: the base set passes every check
    (without a device the launch itself then fails with TD_ERR_CUDA)."""
    cabi = _cabi()
    buf, ptrs, a = _combine_args()
    st = _call_combine(a, ptrs, buf)
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        assert st == cabi.TD_OK, _last_error()
    else:
        assert st == cabi.TD_ERR_CUDA, _last_error()


def _gather_call(n_views, bx, by, H=16, W=1024, s=1, oh=4, ow=4, second=None):
    cabi = _cabi()
    buf = _scratch()
    sec = _i32(second if second is not None else [0] * n_views)
    return cabi.lib.td_dilated_gather(buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), 1, 1, H, W, s, oh, ow, _i32(bx), _i32(by), sec,
                                      n_views, cabi.TD_F16, _stream())


def test_dilated_gather_refuses_65_views():
    st = _gather_call(MAX_VIEWS + 1, [0] * (MAX_VIEWS + 1), [0] * (MAX_VIEWS + 1))
    assert st == _cabi().TD_ERR_INVALID_ARG and _last_error() == "td_dilated_gather: bad arguments"


@pytest.mark.parametrize("bx,by", [(1021, 0), (0, 13), (-1, 0), (0, -1), (1 << 20, 0)], ids=["x_past", "y_past", "x_neg", "y_neg", "x_huge"])
def test_dilated_gather_refuses_views_past_the_canvas(bx, by):
    """A 4x4 view at s = 1 on a 16x1024 canvas: the last column is bx + 3 < 1024, the last row by + 3 < 16."""
    st = _gather_call(2, [0, bx], [0, by])
    assert st == _cabi().TD_ERR_INVALID_ARG and _last_error() == "td_dilated_gather: view 1 out of range"


@pytest.mark.parametrize("k", [0, 2, 14, MAX_KERNEL + 1, MAX_KERNEL + 2, -1])
def test_depthwise_conv_refuses_unsupported_kernels(k):
    cabi = _cabi()
    buf = _scratch()
    taps = (ctypes.c_float * (17 * 17))()
    st = cabi.lib.td_depthwise_conv2d(buf.data_ptr(), buf.data_ptr(), 1, 4, 4, taps, k, cabi.TD_F16, _stream())
    assert st == cabi.TD_ERR_INVALID_ARG and _last_error().startswith("td_depthwise_conv2d: bad arguments")


# ------------------------------------------------------------------------------------------------ td_dilated_gather (GPU)
def _gather(x, x2, views, second, s, oh, ow):
    cabi = _cabi()
    N, C, H, W = x.shape
    out = torch.empty((len(views) * N, C, oh, ow), dtype=x.dtype, device=x.device)
    cabi.check(cabi.lib.td_dilated_gather(x.data_ptr(), x2.data_ptr(), out.data_ptr(), N, C, H, W, s, oh, ow, _i32([v[0] for v in views]),
                                          _i32([v[1] for v in views]), _i32(second), len(views), cabi.dtype_code(x.dtype), _stream()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("s", SCALES)
def test_dilated_gather_is_the_reference_slices(s, dn):
    """All 2 s^2 mixture views of every canvas shape, grid (off 0) and jittered (views at off + (bx, by)), gathered in
    launches of at most 64 views whose source flags are mixed within the launch."""
    dt = DTS[dn]
    rng = np.random.Generator(np.random.PCG64(100 + s))
    for kind in CANVASES:
        for off in (0, 5):
            H, W, end_y, end_x, oh, ow = _canvas(kind, s, off)
            end = W - off
            x = _latent(10 * s + off, (2, 4, H, W), dt).cuda()
            x2 = _latent(10 * s + off + 1, (2, 4, H, W), dt).cuda()
            views = _views(s, True)
            second = [int(v) for v in rng.integers(0, 2, len(views))]
            step = min(MAX_VIEWS, max(1, len(views) - 1))        # the last launch is partial whenever there is more than one
            got = torch.cat([_gather(x, x2, [(bx + off, by + off) for bx, by in views[i:i + step]], second[i:i + step], s, oh, ow)
                             for i in range(0, len(views), step)], dim=0)
            slices = [(x2 if sec else x)[:, :, by + off:end:s, bx + off:end:s] for (bx, by), sec in zip(views, second)]
            assert all(t.shape[2:] == (oh, ow) for t in slices)
            assert torch.equal(got.view(torch.int16 if dt != torch.float32 else torch.int32),
                               torch.cat(slices, dim=0).view(torch.int16 if dt != torch.float32 else torch.int32)), f"{kind} off {off}"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 63, MAX_VIEWS])
def test_dilated_gather_view_count_up_to_the_table_limit(n):
    """1 to 64 views in one launch at s = 8; every view has its own offset and source."""
    s, H, W = 8, 64, 80
    oh, ow = 7, 9
    x = _latent(7, (1, 4, H, W), torch.float16).cuda()
    x2 = _latent(8, (1, 4, H, W), torch.float16).cuda()
    views = [((3 * v) % 16, (5 * v) % 8) for v in range(n)]
    second = [(v * 7 // 3) & 1 for v in range(n)]
    got = _gather(x, x2, views, second, s, oh, ow)
    want = torch.cat([(x2 if sec else x)[:, :, by:by + oh * s:s, bx:bx + ow * s:s] for (bx, by), sec in zip(views, second)], dim=0)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
def test_dilated_gather_offsets_past_255(dn):
    """View offsets >= 256 on a 1024-wide canvas gather from those offsets (they used to be truncated to 8 bits, which
    stays in bounds and reads the wrong pixels)."""
    dt = DTS[dn]
    s, H, W, oh, ow = 3, 520, 1024, 60, 200
    x = _latent(41, (1, 4, H, W), dt).cuda()
    x2 = _latent(42, (1, 4, H, W), dt).cuda()
    views = [(300, 260), (257, 0), (0, 299), (420, 256), (5, 7), (256, 1)]
    second = [0, 1, 0, 1, 1, 0]
    got = _gather(x, x2, views, second, s, oh, ow)
    want = torch.cat([(x2 if sec else x)[:, :, by:by + oh * s:s, bx:bx + ow * s:s] for (bx, by), sec in zip(views, second)], dim=0)
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ combine (GPU)
def _combine(x_local, outs, vpb, n_views, s, oh, ow, off, end_y, end_x, mixture, c2, one_minus_c2):
    cabi = _cabi()
    N, C, H, W = x_local.shape
    res = torch.empty_like(x_local)
    ptrs = (ctypes.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    common = (N, C, H, W, s, oh, ow)
    tail = (end_y, end_x, int(mixture), c2, one_minus_c2, cabi.dtype_code(x_local.dtype), _stream())
    if off:
        cabi.check(cabi.lib.td_demofusion_combine_offset(x_local.data_ptr(), ptrs, len(outs), vpb, n_views, res.data_ptr(), *common, off, *tail))
    else:
        cabi.check(cabi.lib.td_demofusion_combine(x_local.data_ptr(), ptrs, len(outs), vpb, n_views, res.data_ptr(), *common, *tail))
    return res


def _combine_reference(x_local, allv, views, s, off, end, mixture, c2_t):
    """demofusion.py:296-322 as the reference evaluates it: eager ops in the latent dtype on the GPU."""
    N = x_local.shape[0]
    xg = torch.zeros_like(x_local)
    for idx, (bx, by) in enumerate(views):
        xg[:, :, by + off:end:s, bx + off:end:s] += allv[idx * N:(idx + 1) * N]
    if mixture:
        xg = xg / 2
    return x_local * (1 - c2_t) + xg * c2_t


def _combine_fp32(x_local, allv, views, s, off, end, mixture, c2_t):
    """The same expression in fp32 with one final rounding: what a kernel that skipped the per-op rounding would give."""
    return _combine_reference(x_local.float(), allv.float(), views, s, off, end, mixture, c2_t).to(x_local.dtype)


def _check_combine(s, dt, mixture, kind, off, vpb, seed):
    H, W, end_y, end_x, oh, ow = _canvas(kind, s, off)
    N, C = 2, 4
    views = _views(s, mixture)
    n = len(views)
    x_local = _latent(seed, (N, C, H, W), dt).cuda()
    allv = _latent(seed + 1, (n * N, C, oh, ow), dt).cuda()
    outs = [allv[b * vpb * N:min((b + 1) * vpb, n) * N] for b in range(-(-n // vpb))]
    c2_t = odf.cosine_factor(s + 2 * int(mixture), 14) ** 1.0          # 0-dim fp32, as the delegate computes it
    got = _combine(x_local, outs, vpb, n, s, oh, ow, off, end_y, end_x, mixture, float(c2_t), float(1 - c2_t))
    want = _combine_reference(x_local, allv, views, s, off, W - off, mixture, c2_t)
    what = f"s {s} {dt} mixture {mixture} {kind} off {off} vpb {vpb}"
    bits = torch.int32 if dt == torch.float32 else torch.int16
    assert torch.equal(got.view(bits), want.view(bits)), f"{what}: {int((got != want).sum())} elements differ in value"
    if dt != torch.float32:    # the inputs can tell the per-op rounding of the dtype from a single final rounding
        assert not torch.equal(want, _combine_fp32(x_local, allv, views, s, off, W - off, mixture, c2_t)), what
    if kind == "portrait":     # rows past end_y take no view: out = x_local * (1 - c2) there
        assert end_y < H - off


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("mixture", [False, True], ids=["plain", "mixture"])
@pytest.mark.parametrize("s", SCALES)
def test_combine_is_the_eager_reference(s, mixture, dn):
    """td_demofusion_combine (off 0) and td_demofusion_combine_offset (off = jitter range) on landscape, portrait and
    square canvases; views in batches whose last one is partial whenever the view count allows it."""
    n = len(_views(s, mixture))
    vpb = n // 3 + 1 if n > 2 else 1
    for kind in CANVASES:
        for off in (0, 6):
            _check_combine(s, DTS[dn], mixture, kind, off, vpb, seed=1000 + 17 * s + off)


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("off", [0, 6])
def test_combine_128_batch_pointers(off, dn):
    """s = 8, mixture, one view per batch: 128 batch pointers, the table's limit (tile_bs_g = 1 in the UI)."""
    _check_combine(8, DTS[dn], True, "portrait", off, 1, seed=77 + off)


# ------------------------------------------------------------------------------------------------ depthwise conv (GPU)
def _conv(x, taps):
    cabi = _cabi()
    planes = x.shape[0] * x.shape[1]
    k = taps.shape[0]
    out = torch.empty_like(x)
    w = np.ascontiguousarray(taps.float().numpy())
    cabi.check(cabi.lib.td_depthwise_conv2d(x.data_ptr(), out.data_ptr(), planes, x.shape[2], x.shape[3],
                                            w.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), k, cabi.dtype_code(x.dtype), _stream()))
    return out


def _conv64(x, taps):
    """Depthwise zero-padded conv in float64 on the host: (value, sum of |x * w|)."""
    C = x.shape[1]
    w = taps.double()[None, None].repeat(C, 1, 1, 1)
    xd = x.cpu().double()
    k = taps.shape[0]
    return (F.conv2d(xd, w, padding=k // 2, groups=C), F.conv2d(xd.abs(), w.abs(), padding=k // 2, groups=C))


def _neighbours(r: torch.Tensor):
    """r and its two neighbours in r's 16-bit dtype (towards -inf and +inf), as float64."""
    b = r.cpu().contiguous().view(torch.int16).numpy().astype(np.int32) & 0xFFFF
    neg = (b & 0x8000) != 0
    zero_pos, zero_neg = b == 0, b == 0x8000
    up = np.where(neg, b - 1, b + 1)
    down = np.where(neg, b + 1, b - 1)
    up = np.where(zero_neg, 0x0001, up)
    down = np.where(zero_pos, 0x8001, down)

    def back(u):
        return torch.from_numpy(u.astype(np.uint16).view(np.int16)).view(r.dtype).double()
    return r.cpu().double(), back(down), back(up)


def _bound32(absref, k):
    """k^2 roundings of at most 2^-24 relative each, plus half a subnormal step each where the sum underflows."""
    return k * k * (2.0 ** -23 * absref + 2.0 ** -150)


def _conv_violations(got, ref, absref, k, dt):
    """Elements of `got` outside the per-element rounding bound around `ref` (float64)."""
    g = got.cpu().double()
    if dt == torch.float32:
        return int(((g - ref).abs() > _bound32(absref, k)).sum())
    r, lo, hi = _neighbours(ref.to(dt))
    ok = (g == r) | (g == lo) | (g == hi)
    return int((~ok).sum())


def _conv_bound_wrt(got, ref_dt, absref, k, dt):
    """The same bound with a reference already in the dtype (F.conv2d on the GPU)."""
    g, rd = got.cpu().double(), ref_dt.cpu()
    if dt == torch.float32:
        return int(((g - rd.double()).abs() > _bound32(absref, k)).sum())
    r, lo, hi = _neighbours(rd)
    return int((~((g == r) | (g == lo) | (g == hi))).sum())


CONV_SHAPES = [(2, 4, 37, 53), (1, 3, 1, 1), (1, 2, 3, 7), (1, 2, 7, 3), (3, 1, 15, 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("s", SCALES)
def test_depthwise_conv_against_float64(s, dn, monkeypatch):
    """k = 2s - 1 taps: the class's gaussian (rounded to the dtype) and a random asymmetric kernel, on odd canvases
    and on canvases smaller than the kernel (every tap there touches zero padding)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    dt, k = DTS[dn], 2 * s - 1
    sigma = 0.6 * float(0.99 * odf.cosine_factor(3, 14) + 1e-2)
    gauss = DemoFusion.gaussian_kernel(None, k, sigma, 1)[0, 0].to(dt).float()
    g = torch.Generator().manual_seed(s)
    asym = torch.rand((k, k), generator=g, dtype=torch.float64) - 0.3
    asym = (asym / asym.abs().sum()).to(dt).float()
    for taps, name in ((gauss, "gaussian"), (asym, "asymmetric")):
        for si, shape in enumerate(CONV_SHAPES):
            x = _latent(300 + 10 * s + si, shape, dt).cuda()
            got = _conv(x, taps)
            ref, absref = _conv64(x, taps)
            what = f"k {k} {name} {shape} {dt}"
            assert _conv_violations(got, ref, absref, k, dt) == 0, what
            # the reference's own call: F.conv2d in the dtype on the GPU, kernel cast to the dtype (demofusion.py:173-178)
            C = shape[1]
            want_dt = F.conv2d(x, taps.to(dt)[None, None].repeat(C, 1, 1, 1).cuda(), padding=k // 2, groups=C)
            assert _conv_bound_wrt(got, want_dt, absref, k, dt) == 0, what + " vs F.conv2d"
            if name == "asymmetric" and k > 1 and shape[2] >= k and shape[3] >= k:
                # a flipped or transposed tap index would not pass this test
                assert _conv_violations(_conv(x, taps.flip(0, 1)), ref, absref, k, dt) > 0, what + " flipped"
                assert _conv_violations(_conv(x, taps.t().contiguous()), ref, absref, k, dt) > 0, what + " transposed"


# ------------------------------------------------------------------------------------------------ renormalise (GPU)
def _stats_input(case: str, dt):
    """The case's latent on the GPU.  Near-maximum outliers only in fp16: squared in the fp32 statistics, those of bf16
    and fp32 overflow (as they do in torch's own var of a bf16 / fp32 tensor)."""
    big = dt == torch.float16
    if case == "cfg5":                                   # SDXL 6144^2 at the x4 phase: 2x4x768^2
        return _latent(51, (2, 4, 768, 768), dt, near_max=big).cuda()
    if case == "cfg5_jitter":                            # the same, zero-padded by its jitter range (32)
        return F.pad(_latent(52, (2, 4, 768, 768), dt, near_max=big), (32, 32, 32, 32)).cuda()
    if case == "s8_base128":                             # s = 8 of a 128^2 base latent: 2x4x1024^2
        return _latent(53, (2, 4, 1024, 1024), dt, near_max=big).cuda()
    if case == "odd_count":                              # 105105 elements: scalar path
        return _latent(54, (1, 3, 5 * 77, 91), dt, near_max=big).cuda()
    if case == "misaligned":                             # starts one element off 16-byte alignment: scalar path
        return _latent(55, (2 * 4 * 96 * 80 + 1,), dt, near_max=big).cuda()[1:]
    if case == "mean_over_std":                          # |mean| ~ 100 x std
        return (synth.latent(56, (2, 4, 192, 160), torch.float64) * 0.5 + 64.0).to(dt).cuda()
    raise KeyError(case)


STATS_CASES = ["cfg5", "cfg5_jitter", "s8_base128", "odd_count", "misaligned", "mean_over_std"]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("case", STATS_CASES)
def test_whole_tensor_stats_against_float64(case, dn):
    """td_gn_stats with nseg = 1, unbiased = 1 -- what DemoFusion._renormalise reads for g.mean() / g.std()."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    dt = DTS[dn]
    x = _stats_input(case, dt)
    if case == "misaligned":
        assert x.data_ptr() % 16 != 0
    var, mean = tilevae._segment_stats(x, 1, x.numel(), unbiased=True)
    xd = x.double()
    m64, v64 = xd.mean().item(), xd.var(unbiased=True).item()
    m, v = mean.item(), var.item()
    assert abs(m - m64) <= 2e-6 + 2e-5 * abs(m64), f"{case} {dt}: mean {m} vs {m64}"
    assert abs(v - v64) <= 1e-6 + 5e-5 * abs(v64), f"{case} {dt}: var {v} vs {v64}"


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
def test_affine_is_the_eager_renormalise(dn):
    """td_affine_clamp with infinite bounds == (g - m) / sd * so + mo on 0-dim dtype tensors, eager on the GPU."""
    cabi = _cabi()
    dt = DTS[dn]
    g = _latent(61, (2, 4, 72, 88), dt).cuda()
    g[g.abs() > 1e4] = 3.0                       # keep the statistics finite; the subnormals and signed zeros stay
    x = (_latent(62, (2, 4, 72, 88), dt, outliers=False).cuda() * 1.5 + 0.25).to(dt)
    m, sd, mo, so = g.mean(), g.std(), x.mean(), x.std()
    assert m.dim() == 0 and m.dtype == dt
    want = (g - m) / sd * so + mo
    got = g.clone()
    f = lambda t: t.float().reshape(1).contiguous()
    mf, sdf, mof, sof = f(m), f(sd), f(mo), f(so)
    lo = torch.full((1,), -float("inf"), device="cuda")
    hi = torch.full((1,), float("inf"), device="cuda")
    n, c, hh, ww = got.shape
    cabi.check(cabi.lib.td_affine_clamp(got.data_ptr(), n * c, 1, hh * ww, cabi.dtype_code(dt), mf.data_ptr(), sdf.data_ptr(),
                                        mof.data_ptr(), sof.data_ptr(), lo.data_ptr(), hi.data_ptr(), _stream()))
    bits = torch.int32 if dt == torch.float32 else torch.int16
    assert torch.equal(got.view(bits), want.view(bits))


# ------------------------------------------------------------------------------------------------ whole step (GPU)
WINDOW, OVERLAP, TILE_BS, SIG, CS2, CS3, STEP, T_ENC = 24, 12, 4, 0.6, 1.0, 1.0, 3, 14
SEED = 20240922


def _jitter_range(h, w):
    overlap = max(0, min(OVERLAP, WINDOW - 4))
    stride = max(4, WINDOW - overlap)
    return min(max((min(w, h) - stride) // 4, 0), min(int(WINDOW / 2), int(overlap / 2)))


def _step_size(s, kind, jitter):
    """A small latent (h, w) the delegate accepts at scale s: sides multiples of s on the grid; with jitter the
    smallest heights past that for which min(H, W - jr) - jr and W - 2 jr are multiples of s (H, W padded)."""
    a, b = s * math.ceil(48 / s), s * math.ceil(72 / s)
    h, w = (a, b) if kind == "landscape" else (b, a)
    if not jitter:
        return h, w, 0
    for hh in range(h, h + s * s + 1):
        jr = _jitter_range(hh, w)
        H, W = hh + 2 * jr, w + 2 * jr
        if (min(H, W - jr) - jr) % s == 0 and (W - 2 * jr) % s == 0 and jr > 0:
            return hh, w, jr
    raise AssertionError("no accepted size")


def _delegate(s, mixture, jitter, h, w, tile_bs_g):
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    p = types.SimpleNamespace(width=w * 8, height=h * 8, sampler_name="Euler a", current_scale_num=s, mixture=mixture,
                              gaussian_filter=True, random_jitter=jitter, cosine_scale_1=3.0, cosine_scale_2=CS2,
                              cosine_scale_3=CS3, current_step=STEP, steps=20, t_enc=T_ENC, sd_model=None)
    inner = types.SimpleNamespace(forward=None)
    d = DemoFusion(p, types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=inner, image_cfg_scale=None, forward=None)))
    d.window_size, d.sig = WINDOW, SIG
    random.seed(SEED)
    d.get_views(OVERLAP, TILE_BS, tile_bs_g)
    d.sampler_forward = position_aware_denoise(d)
    d.cosine_factor = odf.cosine_factor(STEP, T_ENC)
    return d


STEP_CASES = [(s, kind, jitter) for s in (1, 3, 5, 8) for kind in ("landscape", "portrait") for jitter in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("mixture", [False, True], ids=["plain", "mixture"])
@pytest.mark.parametrize("s,kind,jitter", STEP_CASES, ids=[f"s{s}-{k}-{'jitter' if j else 'grid'}" for s, k, j in STEP_CASES])
def test_sample_one_step_matches_oracle(s, kind, jitter, mixture, dn):
    dt = DTS[dn]
    h, w, jr = _step_size(s, kind, jitter)
    tile_bs_g = 1 if s == 8 else 3
    d = _delegate(s, mixture, jitter, h, w, tile_bs_g)
    assert d.jitter_range == jr
    if s == 8:
        assert d.global_num_batches == (2 * s * s if mixture else s * s)
    N, C = 2, 4
    x = synth.latent(900 + s, (N, C, h, w), dt)
    if jitter:
        local, _, _, jr_o = tiling.demofusion_views_jitter(w, h, WINDOW, OVERLAP, random.Random(SEED))
        assert jr_o == jr
    else:
        local, _, _ = tiling.demofusion_views(w, h, WINDOW, OVERLAP)
    assert [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb] == local
    lb = [local[i * d.tile_bs:(i + 1) * d.tile_bs] for i in range(d.num_batches)]
    views = odf.global_views(s, mixture)
    gb = [views[i * d.global_tile_bs:(i + 1) * d.global_tile_bs] for i in range(d.global_num_batches)]
    xp = F.pad(x, (jr, jr, jr, jr), "constant", value=0) if jr else x
    want = odf.sample_one_step(xp, lb, gb, s, mixture, True, SIG, d.cosine_factor, CS2, CS3,
                               lambda t, b: synth.fake_denoise(t, b, N), lambda t, b: demo_denoise(t), jitter_range=jr)
    cond = {"c_crossattn": [torch.zeros(N, 77, 8, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
    got = d.sample_one_step(xp.cuda(), torch.ones(N, device="cuda"), cond)
    assert got.dtype == dt and got.shape == want.shape
    tol = {torch.float32: 3e-6, torch.float16: 2e-3, torch.bfloat16: 1.6e-2}[dt]
    err = (got.cpu().float() - want.float()).abs().max().item()
    assert err <= tol * max(1.0, want.float().abs().max().item()), f"{h}x{w} jr {jr}: max err {err}"
