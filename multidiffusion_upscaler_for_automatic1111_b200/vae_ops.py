"""Tensor wrappers of the channels-last tiled-VAE kernels (csrc/td_conv.cu, csrc/td_nhwc.cu).

Activations are NHWC fp16 / bf16 tensors `[N, H, W, C]` (contiguous, C innermost); convolution weights are packed once
per network into `[kh*kw, Cout, Cin]` (channels zero-padded to what the implicit GEMM wants).  Every function enqueues
on the current CUDA stream and refuses CPU tensors: there is no fallback.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from ._cabi import TdConvDesc, check, current_stream_ptr, dtype_code, lib

NUM_GROUPS = 32
GN_EPS = 1e-6


def _cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor: the tiled-VAE path has no CPU fallback (got {t.device})")
    if t.dtype not in (torch.float16, torch.bfloat16):
        raise TypeError(f"{what}: the tensor-core path computes in float16 / bfloat16 (got {t.dtype})")


def round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def pack_conv_weight(weight: torch.Tensor, dtype: torch.dtype, cin_pad: Optional[int] = None, cout_pad: Optional[int] = None) -> torch.Tensor:
    """torch conv weight [Cout, Cin, kh, kw] -> [kh*kw, Cout_p, Cin_p] (tap-major, K innermost), zero-padded."""
    co, ci, kh, kw = weight.shape
    cin_p = cin_pad or round_up(ci, 64)
    cout_p = cout_pad or co
    w = torch.zeros((kh * kw, cout_p, cin_p), dtype=dtype, device=weight.device)
    w[:, :co, :ci] = weight.detach().permute(2, 3, 0, 1).reshape(kh * kw, co, ci).to(dtype)
    return w.contiguous()


def fold_upsample_weight(weight: torch.Tensor, dtype: torch.dtype, cin_pad: Optional[int] = None) -> torch.Tensor:
    """3x3 taps of a convolution that follows a nearest-2x upsample, folded for td_upconv2x_nhwc: [Cout, Cin, 3, 3] ->
    [16, Cout, Cin_p].  Output parity py reads low-resolution rows {i-1+py, i+py}; the hi-res rows 2i+py+ky-1 (ky = 0..2)
    that land on the same low-resolution row share one folded tap (summed in fp32, rounded once):
        py = 0: row i-1 <- ky 0        row i   <- ky 1 + ky 2
        py = 1: row i   <- ky 0 + ky 1 row i+1 <- ky 2                    (columns alike)."""
    co, ci, kh, kw = weight.shape
    assert kh == 3 and kw == 3
    cin_p = cin_pad or round_up(ci, 64)
    w32 = weight.detach().float()
    groups = (((0,), (1, 2)), ((0, 1), (2,)))        # [parity][tap] -> 3x3 indices summed
    out = torch.zeros((16, co, cin_p), dtype=dtype, device=weight.device)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    acc = torch.zeros((co, ci), dtype=torch.float32, device=weight.device)
                    for ky in groups[py][ty]:
                        for kx in groups[px][tx]:
                            acc += w32[:, :, ky, kx]
                    out[(py * 2 + px) * 4 + ty * 2 + tx, :, :ci] = acc.to(dtype)
    return out.contiguous()


def _post_stride(post, N: int, Cout: int) -> int:
    """Elements between the images' post vectors: post = (scale, shift, act) with scale / shift [Cout] (one set for every
    image) or [N, >= Cout] (image n's GroupNorm constants in row n)."""
    if post is None:
        return 0
    scale, shift = post[0], post[1]
    assert scale.dtype == torch.float32 and shift.dtype == torch.float32 and scale.shape == shift.shape and scale.is_contiguous() and shift.is_contiguous()
    if scale.dim() == 1 or scale.shape[0] == 1:
        assert scale.numel() >= Cout
        return 0
    assert scale.dim() == 2 and scale.shape[0] == N and scale.shape[1] >= Cout, f"post constants {tuple(scale.shape)} for {N} images"
    return scale.stride(0)


def upconv2x_nhwc(x: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor] = None, *, cout: Optional[int] = None,
                  out: Optional[torch.Tensor] = None, post: Optional[Tuple[torch.Tensor, torch.Tensor, bool]] = None, dual: bool = False):
    """Nearest-2x upsample + 3x3 / pad 1 convolution in one pass over the LOW-resolution x [N, H, W, Cin] ->
    [N, 2H, 2W, Cout]; w16 from fold_upsample_weight.  post as in conv2d_nhwc; dual (needs post): returns (result before
    post, result after post)."""
    _cuda(x, "x"); _cuda(w16, "w16")
    N, H, W, Cin = x.shape
    taps, cout_rows, w_cin = w16.shape
    assert taps == 16 and w_cin == Cin and x.is_contiguous() and w16.is_contiguous()
    Cout = cout or cout_rows
    if out is None:
        out = torch.empty((N, 2 * H, 2 * W, Cout), dtype=x.dtype, device=x.device)
    assert out.is_contiguous() and out.shape == (N, 2 * H, 2 * W, Cout)
    d = TdConvDesc(N=N, H=H, W=W, Cin=Cin, Cout=Cout, kh=3, kw=3, stride=1, pad_top=1, pad_left=1, OH=2 * H, OW=2 * W,
                   dtype=dtype_code(x.dtype), bias_per_row=0, alpha=1.0, x_pitch=x.stride(2), w_pitch=w16.stride(1), y_pitch=out.stride(2),
                   res_pitch=0, post_scale=post[0].data_ptr() if post is not None else None,
                   post_shift=post[1].data_ptr() if post is not None else None, post_act=int(bool(post[2])) if post is not None else 0,
                   post_stride=_post_stride(post, N, Cout))
    out2 = None
    if dual:
        assert post is not None, "the second output is the post stage's result"
        out2 = torch.empty_like(out)
        d.y2, d.y2_pitch = out2.data_ptr(), out2.stride(2)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_cuda
    with torch.cuda.device(x.device):
        check(lib.td_upconv2x_nhwc(ctypes.byref(d), x.data_ptr(), w16.data_ptr(), bias.data_ptr() if bias is not None else None,
                                   out.data_ptr(), current_stream_ptr(x.device)))
    return (out, out2) if dual else out


def conv2d_nhwc(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, ksize: int, stride: int = 1,
                pad: Tuple[int, int] = (0, 0), out_hw: Optional[Tuple[int, int]] = None, residual: Optional[torch.Tensor] = None,
                alpha: float = 1.0, cout: Optional[int] = None, out: Optional[torch.Tensor] = None,
                bias_per_row: bool = False, post: Optional[Tuple[torch.Tensor, torch.Tensor, bool]] = None, dual: bool = False):
    """One convolution on the tensor cores.  x: [N, H, W, Cin] NHWC; w: packed [ksize*ksize, Cout_rows, Cin];
    bias: fp32 [Cout] (or [N*OH*OW] with bias_per_row); residual: [N, OH, OW, Cout] added in the epilogue.
    pad = (top, left) zero padding; out_hw defaults to the 'same' size for stride 1.
    post = (scale, shift, silu): per-channel affine (+ SiLU) on the fp32 result, scale / shift fp32 [Cout] for every image
    or [N, Cout] per image; dual (needs post): two outputs, returns (result before post, result after post)."""
    _cuda(x, "x"); _cuda(w, "w")
    N, H, W, Cin = x.shape
    taps, cout_rows, w_cin = w.shape
    assert taps == ksize * ksize and w_cin == Cin, f"weight {tuple(w.shape)} does not match ksize {ksize} / Cin {Cin}"
    Cout = cout or cout_rows
    # the kernel steps from one tap's weights to the next by Cout rows (include/td_b200.h: w is [kh*kw][Cout][w_pitch]):
    # a 3x3 weight packed with more rows than Cout would be read at the wrong tap offsets
    assert Cout <= cout_rows and (taps == 1 or Cout == cout_rows), f"Cout {Cout} vs {cout_rows} weight rows per tap ({taps} taps)"
    OH, OW = out_hw if out_hw is not None else (H, W)
    if out is None:
        out = torch.empty((N, OH, OW, Cout), dtype=x.dtype, device=x.device)
    d = TdConvDesc(N=N, H=H, W=W, Cin=Cin, Cout=Cout, kh=ksize, kw=ksize, stride=stride, pad_top=pad[0], pad_left=pad[1],
                   OH=OH, OW=OW, dtype=dtype_code(x.dtype), bias_per_row=int(bias_per_row), alpha=float(alpha),
                   x_pitch=x.stride(2), w_pitch=w.stride(1), y_pitch=out.stride(2),
                   res_pitch=residual.stride(2) if residual is not None else 0,
                   post_scale=post[0].data_ptr() if post is not None else None, post_shift=post[1].data_ptr() if post is not None else None,
                   post_act=int(bool(post[2])) if post is not None else 0, post_stride=_post_stride(post, N, Cout))
    assert x.stride(3) == 1 and out.stride(3) == 1 and w.stride(2) == 1
    out2 = None
    if dual:
        assert post is not None, "the second output is the post stage's result"
        out2 = torch.empty_like(out)
        d.y2, d.y2_pitch = out2.data_ptr(), out2.stride(2)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_cuda
    with torch.cuda.device(x.device):
        check(lib.td_conv2d_nhwc(ctypes.byref(d), x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                 residual.data_ptr() if residual is not None else None, out.data_ptr(), current_stream_ptr(x.device)))
    return (out, out2) if dual else out


def gemm_nt(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor] = None, alpha: float = 1.0, n: Optional[int] = None,
            out: Optional[torch.Tensor] = None, bias_per_row: bool = False) -> torch.Tensor:
    """D[M, n] = alpha * A[M, K] @ B[n, K]^T (+ bias).  A / B / D are 2-D views with unit inner stride; row pitches
    must be multiples of 8 elements; K a multiple of 64 (out-of-range K of a wider pitch must be zeros)."""
    _cuda(a, "a"); _cuda(b, "b")
    M, K = a.shape
    nb = n or b.shape[0]
    if out is None:
        out = torch.empty((M, round_up(nb, 8)), dtype=a.dtype, device=a.device)[:, :nb]
    d = TdConvDesc(N=1, H=1, W=M, Cin=K, Cout=nb, kh=1, kw=1, stride=1, pad_top=0, pad_left=0, OH=1, OW=M, dtype=dtype_code(a.dtype),
                   bias_per_row=int(bias_per_row), alpha=float(alpha), x_pitch=a.stride(0), w_pitch=b.stride(0), y_pitch=out.stride(0),
                   res_pitch=0)
    with torch.cuda.device(a.device):
        check(lib.td_conv2d_nhwc(ctypes.byref(d), a.data_ptr(), b.data_ptr(), bias.data_ptr() if bias is not None else None, None,
                                 out.data_ptr(), current_stream_ptr(a.device)))
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, alpha: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """O[T, C] = softmax(alpha * Q K^T) V in one fused kernel (csrc/td_attn.cu): online softmax, nothing of size T x T is
    allocated.  q / k / v / out: [T, C] views with unit inner stride, row pitches multiples of 8 elements; C % 64 == 0,
    C <= 512.  [N, T, C] views: N images in one launch (td_attention_batched), image strides multiples of 8 elements."""
    _cuda(q, "q"); _cuda(k, "k"); _cuda(v, "v")
    shape = tuple(q.shape)
    assert len(shape) in (2, 3) and k.shape == shape and v.shape == shape, f"q {shape}, k {tuple(k.shape)}, v {tuple(v.shape)} differ"
    assert k.dtype == q.dtype and v.dtype == q.dtype and k.device == q.device and v.device == q.device
    if out is None:
        out = torch.empty(shape, dtype=q.dtype, device=q.device)
    assert out.shape == shape and out.dtype == q.dtype
    for name, t in (("q", q), ("k", k), ("v", v), ("out", out)):
        assert t.stride(-1) == 1 and t.stride(-2) % 8 == 0, f"{name}: unit inner stride and a row pitch that is a multiple of 8 (got {t.stride()})"
    T, C = shape[-2:]
    with torch.cuda.device(q.device):
        if len(shape) == 2:
            check(lib.td_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), T, C, q.stride(0), k.stride(0), v.stride(0),
                                   out.stride(0), float(alpha), dtype_code(q.dtype), current_stream_ptr(q.device)))
        else:
            check(lib.td_attention_batched(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), shape[0], T, C, q.stride(1), k.stride(1),
                                           v.stride(1), out.stride(1), q.stride(0), k.stride(0), v.stride(0), out.stride(0), float(alpha),
                                           dtype_code(q.dtype), current_stream_ptr(q.device)))
    return out


def nchw_to_nhwc(x: torch.Tensor, cpad: int) -> torch.Tensor:
    """[N, C, h, w] view (unit inner stride) -> contiguous [N, h, w, cpad], channels zero-padded."""
    _cuda(x, "x")
    N, C, h, w = x.shape
    assert x.stride(3) == 1
    y = torch.empty((N, h, w, cpad), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.td_nchw_to_nhwc(x.data_ptr(), y.data_ptr(), N, C, h, w, x.stride(0), x.stride(1), x.stride(2), cpad, dtype_code(x.dtype),
                                  current_stream_ptr(x.device)))
    return y


def nchw_to_nhwc_wrap(z: torch.Tensor, bbox, cpad: int) -> torch.Tensor:
    """Tile [x1, x2) x [y1, y2) of a periodic canvas z [N, C, H, W] (contiguous), bounds in unwrapped coordinates (they may
    be negative or pass the canvas) -> contiguous [N, y2 - y1, x2 - x1, cpad], channels zero-padded."""
    _cuda(z, "z")
    N, C, H, W = z.shape
    assert z.is_contiguous()
    x1, x2, y1, y2 = (int(v) for v in bbox)
    y = torch.empty((N, y2 - y1, x2 - x1, cpad), dtype=z.dtype, device=z.device)
    with torch.cuda.device(z.device):
        check(lib.td_nchw_to_nhwc_wrap(z.data_ptr(), y.data_ptr(), N, C, y2 - y1, x2 - x1, y1, x1, H, W, z.stride(0), z.stride(1), z.stride(2),
                                       cpad, dtype_code(z.dtype), current_stream_ptr(z.device)))
    return y


def nhwc_to_nchw_region(x: torch.Tensor, dst: torch.Tensor, channels: int) -> None:
    """dst[n, c, i, j] = x[n, i, j, c] for c < channels; x: NHWC view [N, rows, cols, >=channels] (unit channel stride),
    dst: NCHW view [N, channels, rows, cols] (unit inner stride)."""
    _cuda(x, "x"); _cuda(dst, "dst")
    N, rows, cols, _ = x.shape
    assert dst.shape == (N, channels, rows, cols) and dst.stride(3) == 1 and x.stride(3) == 1 and x.dtype == dst.dtype
    assert x.stride(1) % x.stride(2) == 0
    with torch.cuda.device(x.device):
        check(lib.td_nhwc_to_nchw_region(x.data_ptr(), dst.data_ptr(), N, channels, rows, cols, x.stride(0), x.stride(1) // x.stride(2),
                                         x.stride(2), dst.stride(0), dst.stride(1), dst.stride(2), dtype_code(x.dtype),
                                         current_stream_ptr(x.device)))


def upsample2x_nhwc(x: torch.Tensor) -> torch.Tensor:
    _cuda(x, "x")
    N, H, W, C = x.shape
    assert x.is_contiguous()
    y = torch.empty((N, 2 * H, 2 * W, C), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.td_upsample2x_nhwc(x.data_ptr(), y.data_ptr(), N, H, W, C, dtype_code(x.dtype), current_stream_ptr(x.device)))
    return y


def gn_stats_nhwc(x: torch.Tensor, groups: int = NUM_GROUPS):
    """Biased variance and mean per (image, group) of channels-last images [N, H, W, C] -> (var, mean) fp32 [N * groups].
    Each image gets the bits of its own one-image reduction (td_gn_stats_nhwc_batched)."""
    _cuda(x, "x")
    assert x.is_contiguous()
    N, H, W, C = x.shape
    dev = x.device
    ws_bytes = lib.td_gn_stats_nhwc_batched_workspace_bytes(N, H * W, C, groups)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    mean = torch.empty(N * groups, dtype=torch.float32, device=dev)
    var = torch.empty(N * groups, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.td_gn_stats_nhwc_batched(x.data_ptr(), N, H * W, C, groups, dtype_code(x.dtype), ws.data_ptr(), ws_bytes, mean.data_ptr(),
                                           var.data_ptr(), current_stream_ptr(dev)))
    return var, mean


def gn_apply_nhwc(x: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor],
                  act: bool, groups: int = NUM_GROUPS, eps: float = GN_EPS, inplace: bool = False) -> torch.Tensor:
    """GroupNorm (+ SiLU) of channels-last images [N, H, W, C] with per-image statistics mean / var fp32 [N * groups]."""
    _cuda(x, "x")
    assert x.is_contiguous()
    N, H, W, C = x.shape
    assert mean.numel() == N * groups and var.numel() == N * groups, f"statistics of {mean.numel()} groups for {N} images"
    assert mean.dtype == torch.float32 and var.dtype == torch.float32 and mean.is_contiguous() and var.is_contiguous()
    y = x if inplace else torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.td_gn_apply_nhwc_batched(x.data_ptr(), y.data_ptr(), N, H * W, C, groups, dtype_code(x.dtype), mean.data_ptr(),
                                           var.data_ptr(), gamma.data_ptr() if gamma is not None else None,
                                           beta.data_ptr() if beta is not None else None, float(eps), int(act),
                                           current_stream_ptr(x.device)))
    return y


def softmax_rows(x: torch.Tensor, cols: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Row softmax over the first `cols` columns of a [rows, pitch] matrix (pitch % 8 == 0); the padding columns get 0."""
    _cuda(x, "x")
    rows, pitch = x.shape
    assert x.is_contiguous()
    y = out if out is not None else torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.td_softmax_rows(x.data_ptr(), y.data_ptr(), rows, cols, pitch, dtype_code(x.dtype), current_stream_ptr(x.device)))
    return y
