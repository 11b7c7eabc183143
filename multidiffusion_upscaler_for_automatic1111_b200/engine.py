"""Tensor-level wrappers over the C-ABI kernels (device pointers + current stream).

PyTorch is plumbing here: it owns the memory and the stream; every byte of the
hot path moves through the hand-written sm_90a kernels in csrc/.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np
import torch

from ._cabi import TD_WRAP_X, TD_WRAP_Y, TdGrid, check, current_stream_ptr, dtype_code, lib

WRAP_X, WRAP_Y = TD_WRAP_X, TD_WRAP_Y   # `wrap` bits of make_grid: the canvas is periodic in x / in y (seamless tiling)


def make_grid(w: int, h: int, tile_w: int, tile_h: int, overlap: int, tile_bs: int, wrap: int = 0) -> TdGrid:
    """init_grid_bbox bookkeeping (abstractdiffusion.py:172-186) -> td_grid.

    `wrap` (WRAP_X | WRAP_Y) tiles those axes as a circle: tiles may run past the canvas edge and continue at 0, so the
    blend mixes both sides of the seam.  The plan records it (`g.wrap`) and every kernel entry reads it from there."""
    g = TdGrid()
    check(lib.td_grid_init(ctypes.byref(g), int(w), int(h), int(tile_w), int(tile_h), int(overlap), int(tile_bs), int(wrap)))
    return g


def grid_bboxes_xywh(g: TdGrid) -> np.ndarray:
    """int32 [T,4] (x, y, w, h) in tile-list order (row outer, col inner)."""
    xs = np.ctypeslib.as_array(g.xs)[:g.cols]
    ys = np.ctypeslib.as_array(g.ys)[:g.rows]
    out = np.empty((g.rows, g.cols, 4), dtype=np.int32)
    out[..., 0] = xs[None, :]
    out[..., 1] = ys[:, None]
    out[..., 2] = g.tile_w
    out[..., 3] = g.tile_h
    return out.reshape(-1, 4)


def scaled_grid(g: TdGrid, scale: int) -> TdGrid:
    """The same tile plan in a space `scale` times finer: pixel-space side inputs (ControlNet hints, x8) are cropped
    with the latent tile list multiplied by opt_f (abstractdiffusion.py:499)."""
    s = TdGrid.from_buffer_copy(g)
    s.H, s.W = g.H * scale, g.W * scale
    s.tile_h, s.tile_w, s.overlap = g.tile_h * scale, g.tile_w * scale, g.overlap * scale
    for i in range(g.rows):
        s.ys[i] = g.ys[i] * scale
    for i in range(g.cols):
        s.xs[i] = g.xs[i] * scale
    return s


def grid_weights(g: TdGrid, tile_weights: Optional[np.ndarray] = None) -> np.ndarray:
    """fp32 [H, W] host weight canvas (utils.py:167,175)."""
    out = np.empty((g.H, g.W), dtype=np.float32)
    tw_ptr = None
    if tile_weights is not None:
        tile_weights = np.ascontiguousarray(tile_weights, dtype=np.float32)
        if tile_weights.shape != (g.tile_h, g.tile_w):
            raise ValueError(f"tile_weights shape {tile_weights.shape} != tile {(g.tile_h, g.tile_w)}")
        tw_ptr = tile_weights.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    check(lib.td_grid_weights(ctypes.byref(g), tw_ptr, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float))))
    return out


def rescale_factor(weights: np.ndarray) -> np.ndarray:
    """1 / weights in fp32 (mixtureofdiffusers.py:32)."""
    weights = np.ascontiguousarray(weights, dtype=np.float32)
    out = np.empty_like(weights)
    check(lib.td_rescale_factor(weights.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), weights.size))
    return out


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor: this path has no CPU fallback (got device {t.device})")


def scatter_tiles(g: TdGrid, x: torch.Tensor, out: Optional[torch.Tensor] = None, tile_begin: int = 0,
                  tile_end: Optional[int] = None, flags: int = 0) -> torch.Tensor:
    """x [N,C,H,W] -> tiles [(tile_end-tile_begin)*N, C, th, tw], tile-major (multidiffusion.py:155)."""
    _require_cuda(x, "x")
    if x.dim() != 4 or x.shape[2] != g.H or x.shape[3] != g.W:
        raise ValueError(f"x shape {tuple(x.shape)} does not match the grid canvas {(g.H, g.W)}")
    x = x.contiguous()
    N, C = x.shape[0], x.shape[1]
    tile_end = g.num_tiles if tile_end is None else tile_end
    shape = ((tile_end - tile_begin) * N, C, g.tile_h, g.tile_w)
    if out is None or tuple(out.shape) != shape or out.dtype != x.dtype or out.device != x.device:
        out = torch.empty(shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.td_scatter_tiles(ctypes.byref(g), x.data_ptr(), out.data_ptr(), N, C, dtype_code(x.dtype),
                                   int(tile_begin), int(tile_end), int(flags), current_stream_ptr(x.device)))
    return out


def _batch_table(g: TdGrid, batch_outs: Sequence[torch.Tensor], N: int, C: int, tile_bs: int):
    if len(batch_outs) == 0:
        raise ValueError("no tile outputs to blend")
    dt = batch_outs[0].dtype
    keep = []
    for b, t in enumerate(batch_outs):
        _require_cuda(t, "tile output")
        n_tiles = min(tile_bs, g.num_tiles - b * tile_bs)
        want = (n_tiles * N, C, g.tile_h, g.tile_w)
        if tuple(t.shape) != want:
            raise ValueError(f"tile batch {b} has shape {tuple(t.shape)}, expected {want}")
        if t.dtype != dt:
            t = t.to(dt)
        keep.append(t.contiguous())
    ptrs = (ctypes.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
    return ptrs, keep, dt


def _fit_batch_table(g: TdGrid, batch_outs: Sequence[torch.Tensor], tile_bs: int):
    """The kernels take at most TD_MAX_BATCH_PTRS output tensors per launch (pointers travel in the kernel parameter
    block).  The reference accepts any batch count (e.g. 441 tiles with tile_bs 3 = 147 batches): concatenate groups of
    k consecutive full batches into one tensor each and report the new tile_bs = k * tile_bs.  Tile order is unchanged."""
    from ._cabi import TD_MAX_BATCH_PTRS
    n = len(batch_outs)
    if n <= TD_MAX_BATCH_PTRS:
        return list(batch_outs), tile_bs
    k = -(-n // TD_MAX_BATCH_PTRS)
    merged = [torch.cat(list(batch_outs[i:i + k]), dim=0) for i in range(0, n, k)]
    return merged, tile_bs * k


def blend_multidiffusion(g: TdGrid, batch_outs: Sequence[torch.Tensor], N: int, C: int, tile_bs: int,
                         weights: torch.Tensor, acc_dtype: torch.dtype, x_buffer: Optional[torch.Tensor] = None,
                         flags: int = 0, out: Optional[torch.Tensor] = None, rcp_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Fused multidiffusion.py:166-167 + :208.  Returns fp32 [N,C,H,W] (fresh unless `out` is given).

    rcp_weights (see `exact_reciprocals`) enables the 3-instruction exact divide for integer weights."""
    batch_outs, tile_bs = _fit_batch_table(g, batch_outs, tile_bs)
    ptrs, keep, tdt = _batch_table(g, batch_outs, N, C, tile_bs)
    dev = keep[0].device
    x_out = out if out is not None else torch.empty((N, C, g.H, g.W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.td_blend_multidiffusion(ctypes.byref(g), ptrs, len(keep), int(tile_bs), N, C, dtype_code(tdt),
                                          dtype_code(acc_dtype), weights.data_ptr(),
                                          rcp_weights.data_ptr() if rcp_weights is not None else None, x_out.data_ptr(),
                                          x_buffer.data_ptr() if x_buffer is not None else None, int(flags),
                                          current_stream_ptr(dev)))
    return x_out


def exact_reciprocals(weights_host: np.ndarray) -> Optional[np.ndarray]:
    """RN(1/w) for a weight canvas whose entries are all integers in [0, 4096] (MultiDiffusion's
    uniform counts), else None: the precondition of td_blend_multidiffusion's fast exact divide."""
    w = np.ascontiguousarray(weights_host, dtype=np.float32)
    if not (np.all(w == np.floor(w)) and w.min() >= 0 and w.max() <= 4096):
        return None
    with np.errstate(divide="ignore"):
        return rescale_factor(w)


def blend_mixture(g: TdGrid, batch_outs: Sequence[torch.Tensor], N: int, C: int, tile_bs: int,
                  tile_weights: torch.Tensor, rescale: torch.Tensor, x_buffer: torch.Tensor, flags: int = 0) -> torch.Tensor:
    """mixtureofdiffusers.py:122-126; writes and returns x_buffer."""
    batch_outs, tile_bs = _fit_batch_table(g, batch_outs, tile_bs)
    ptrs, keep, tdt = _batch_table(g, batch_outs, N, C, tile_bs)
    dev = keep[0].device
    with torch.cuda.device(dev):
        check(lib.td_blend_mixture(ctypes.byref(g), ptrs, len(keep), int(tile_bs), N, C, dtype_code(tdt),
                                   dtype_code(x_buffer.dtype), tile_weights.data_ptr(), rescale.data_ptr(),
                                   x_buffer.data_ptr(), int(flags), current_stream_ptr(dev)))
    return x_buffer


def blend_mixture_rows(g: TdGrid, band_ptrs: Sequence[int], N: int, C: int, tile_dtype: torch.dtype, tile_weights: torch.Tensor,
                       rescale: torch.Tensor, x_buffer: torch.Tensor, row_begin: int, row_end: int, wait=None,
                       own_bands=(0, 0), flags: int = 0) -> torch.Tensor:
    """`blend_mixture` of the canvas rows [row_begin, row_end) only (row-strip shard), written into those rows of the
    whole-canvas x_buffer; returns it.  band_ptrs: one device pointer per tile ROW (the tiles of row i, [cols*N, C, th, tw]).
    wait: (flags pointer, count, value pointer) -- the CTAs whose tiles leave the own bands [own_bands) first wait until
    flags[0 .. count) >= *value (td_blend_mixture_rows)."""
    _require_cuda(x_buffer, "x_buffer")
    fptr, count, vptr = wait if wait is not None else (None, 0, None)
    ptrs = (ctypes.c_void_p * len(band_ptrs))(*band_ptrs)
    with torch.cuda.device(x_buffer.device):
        check(lib.td_blend_mixture_rows(ctypes.byref(g), ptrs, len(band_ptrs), int(g.cols), N, C, dtype_code(tile_dtype),
                                        dtype_code(x_buffer.dtype), tile_weights.data_ptr(), rescale.data_ptr(), x_buffer.data_ptr(),
                                        int(row_begin), int(row_end), fptr if count else None, int(count), vptr if count else None,
                                        int(own_bands[0]), int(own_bands[1]), int(flags), current_stream_ptr(x_buffer.device)))
    return x_buffer


def blend_multidiffusion_wrap_rows(g: TdGrid, band_ptrs: Sequence[int], N: int, C: int, tile_dtype: torch.dtype, weights: torch.Tensor,
                                   x_out: torch.Tensor, row_begin: int, row_end: int, x_buffer: Optional[torch.Tensor] = None,
                                   wait=None, own_bands=(0, 0), flags: int = 0, tile_bs: Optional[int] = None) -> torch.Tensor:
    """`blend_multidiffusion` of the canvas rows [row_begin, row_end) of a periodic plan (g.wrap != 0) into those rows of the
    fp32 x_out (and of x_buffer, the tile dtype, when given); returns x_out.  band_ptrs / wait / own_bands as in
    `blend_mixture_rows`; `tile_bs` (default g.cols: one pointer per tile row) for another pointer table
    (td_blend_multidiffusion_wrap_rows)."""
    _require_cuda(x_out, "x_out")
    fptr, count, vptr = wait if wait is not None else (None, 0, None)
    ptrs = (ctypes.c_void_p * len(band_ptrs))(*band_ptrs)
    with torch.cuda.device(x_out.device):
        check(lib.td_blend_multidiffusion_wrap_rows(ctypes.byref(g), ptrs, len(band_ptrs), int(g.cols if tile_bs is None else tile_bs), N, C,
                                                    dtype_code(tile_dtype), dtype_code(tile_dtype), weights.data_ptr(), x_out.data_ptr(),
                                                    x_buffer.data_ptr() if x_buffer is not None else None, int(row_begin), int(row_end),
                                                    fptr if count else None, int(count), vptr if count else None, int(own_bands[0]),
                                                    int(own_bands[1]), int(flags), current_stream_ptr(x_out.device)))
    return x_out


def blend_mixture_wrap_rows(g: TdGrid, band_ptrs: Sequence[int], N: int, C: int, tile_dtype: torch.dtype, tile_weights: torch.Tensor,
                            rescale: torch.Tensor, x_buffer: torch.Tensor, row_begin: int, row_end: int, wait=None,
                            own_bands=(0, 0), flags: int = 0) -> torch.Tensor:
    """`blend_mixture_rows` on a periodic plan (g.wrap != 0): td_blend_mixture_wrap_rows."""
    _require_cuda(x_buffer, "x_buffer")
    fptr, count, vptr = wait if wait is not None else (None, 0, None)
    ptrs = (ctypes.c_void_p * len(band_ptrs))(*band_ptrs)
    with torch.cuda.device(x_buffer.device):
        check(lib.td_blend_mixture_wrap_rows(ctypes.byref(g), ptrs, len(band_ptrs), int(g.cols), N, C, dtype_code(tile_dtype),
                                             dtype_code(x_buffer.dtype), tile_weights.data_ptr(), rescale.data_ptr(), x_buffer.data_ptr(),
                                             int(row_begin), int(row_end), fptr if count else None, int(count), vptr if count else None,
                                             int(own_bands[0]), int(own_bands[1]), int(flags), current_stream_ptr(x_buffer.device)))
    return x_buffer


# ---------------------------------------------------------------------------------------------------------
# DemoFusion (tile_methods/demofusion.py): thin wrappers over the C-ABI, one launch each
# ---------------------------------------------------------------------------------------------------------
def dilated_gather(x: torch.Tensor, x_second: Optional[torch.Tensor], view_bx: Sequence[int], view_by: Sequence[int],
                   view_second: Sequence[int], s: int, out_h: int, out_w: int) -> torch.Tensor:
    """demofusion.py:283-308: out[(v*N+n), c, i, j] = src_v[n, c, by_v + i*s, bx_v + j*s]; src_v = x_second where
    view_second[v] else x."""
    _require_cuda(x, "x")
    N, C, H, W = x.shape
    n = len(view_bx)
    out = torch.empty((n * N, C, out_h, out_w), dtype=x.dtype, device=x.device)
    arr = lambda v: (ctypes.c_int32 * n)(*[int(i) for i in v])
    with torch.cuda.device(x.device):
        check(lib.td_dilated_gather(x.data_ptr(), x_second.data_ptr() if x_second is not None else None, out.data_ptr(), N, C, H, W,
                                    int(s), int(out_h), int(out_w), arr(view_bx), arr(view_by), arr(view_second), n,
                                    dtype_code(x.dtype), current_stream_ptr(x.device)))
    return out


def demofusion_combine(x_local: torch.Tensor, view_outs: Sequence[torch.Tensor], views_per_batch: int, n_views: int, s: int,
                       out_h: int, out_w: int, offset: int, end_y: int, end_x: int, mixture: bool, c2: float,
                       one_minus_c2: float) -> torch.Tensor:
    """demofusion.py:296-322 in one launch: strided add-back of the view outputs (in view order, rounded through the
    dtype), `/ 2` in mixture mode, out = x_local*(1-c2) + x_global*c2.  `offset` = jitter_range (0: td_demofusion_combine)."""
    _require_cuda(x_local, "x_local")
    N, C, H, W = x_local.shape
    dev, dt = x_local.device, x_local.dtype
    out = torch.empty_like(x_local)
    ptrs = (ctypes.c_void_p * len(view_outs))(*[t.data_ptr() for t in view_outs])
    with torch.cuda.device(dev):
        if offset:
            check(lib.td_demofusion_combine_offset(x_local.data_ptr(), ptrs, len(view_outs), int(views_per_batch), int(n_views),
                                                   out.data_ptr(), N, C, H, W, int(s), int(out_h), int(out_w), int(offset), int(end_y),
                                                   int(end_x), int(bool(mixture)), c2, one_minus_c2, dtype_code(dt),
                                                   current_stream_ptr(dev)))
        else:
            check(lib.td_demofusion_combine(x_local.data_ptr(), ptrs, len(view_outs), int(views_per_batch), int(n_views), out.data_ptr(),
                                            N, C, H, W, int(s), int(out_h), int(out_w), int(end_y), int(end_x), int(bool(mixture)), c2,
                                            one_minus_c2, dtype_code(dt), current_stream_ptr(dev)))
    return out


def scatter_bboxes(x: torch.Tensor, origins_dev: torch.Tensor, origins_host, n_tiles: int, tile_h: int, tile_w: int,
                   out: Optional[torch.Tensor] = None, wrap: int = 0) -> torch.Tensor:
    """Window LIST scatter (DemoFusion random jitter, demofusion.py:256): tiles[(t*N+n), c] = x[n, c, window t].

    `wrap` (WRAP_X | WRAP_Y, seamless DemoFusion): windows read (o + u) mod L on those axes and zeros off the canvas on the
    others (td_scatter_bboxes_wrap; origins_host is then required)."""
    _require_cuda(x, "x")
    N, C, H, W = x.shape
    shape = (n_tiles * N, C, tile_h, tile_w)
    if out is None or tuple(out.shape) != shape or out.dtype != x.dtype or out.device != x.device:
        out = torch.empty(shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        if wrap:
            check(lib.td_scatter_bboxes_wrap(x.data_ptr(), out.data_ptr(), origins_dev.data_ptr(), origins_host, int(n_tiles), N, C, H, W,
                                             int(tile_h), int(tile_w), int(wrap), dtype_code(x.dtype), current_stream_ptr(x.device)))
        else:
            check(lib.td_scatter_bboxes(x.data_ptr(), out.data_ptr(), origins_dev.data_ptr(), origins_host, int(n_tiles), N, C, H, W,
                                        int(tile_h), int(tile_w), dtype_code(x.dtype), current_stream_ptr(x.device)))
    return out


def blend_bboxes(batch_outs: Sequence[torch.Tensor], tile_bs: int, origins_dev: torch.Tensor, origins_host, n_tiles: int, N: int, C: int,
                 H: int, W: int, tile_h: int, tile_w: int, wrap: int = 0) -> torch.Tensor:
    """Window LIST count-normalised blend (demofusion.py:259-264): fp32 [N,C,H,W] = ordered sum (rounded through the tile
    dtype per add) / max(count, 1).  `wrap` as in `scatter_bboxes`: coverage is modular on those axes, and window pixels
    off the canvas on a bounded axis are dropped (td_blend_bboxes_wrap)."""
    dev, dt = batch_outs[0].device, batch_outs[0].dtype
    _require_cuda(batch_outs[0], "tile output")
    ptrs = (ctypes.c_void_p * len(batch_outs))(*[t.data_ptr() for t in batch_outs])
    out = torch.empty((N, C, H, W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        if wrap:
            check(lib.td_blend_bboxes_wrap(ptrs, len(batch_outs), int(tile_bs), origins_dev.data_ptr(), origins_host, int(n_tiles), N, C, H,
                                           W, int(tile_h), int(tile_w), int(wrap), dtype_code(dt), out.data_ptr(), current_stream_ptr(dev)))
        else:
            check(lib.td_blend_bboxes(ptrs, len(batch_outs), int(tile_bs), origins_dev.data_ptr(), origins_host, int(n_tiles), N, C, H, W,
                                      int(tile_h), int(tile_w), dtype_code(dt), out.data_ptr(), current_stream_ptr(dev)))
    return out



def _region_table(xb: torch.Tensor, regions: Sequence[tuple]):
    """td_region array of `regions` [(x, y, w, h, mode, region_out [N,C,h,w], aux fp32 [h,w] or None)] + the tensors it points at."""
    from ._cabi import TdRegion
    N, C = xb.shape[0], xb.shape[1]
    arr = (TdRegion * max(1, len(regions)))()
    keep = []
    for i, (rx, ry, rw, rh, mode, r_out, aux) in enumerate(regions):
        _require_cuda(r_out, "region output")
        ro = r_out.to(xb.dtype).contiguous()
        if tuple(ro.shape) != (N, C, rh, rw):
            raise ValueError(f"region {i}: output shape {tuple(ro.shape)} != {(N, C, rh, rw)}")
        ax = None
        if aux is not None:
            ax = aux.to(device=xb.device, dtype=torch.float32).expand(rh, rw).contiguous() if aux.dim() == 2 else \
                aux.to(device=xb.device, dtype=torch.float32).reshape(rh, rw).contiguous()
        keep += [ro, ax]
        arr[i] = TdRegion(int(rx), int(ry), int(rw), int(rh), int(mode), ro.data_ptr(), ax.data_ptr() if ax is not None else None)
    return arr, keep


def region_composite(x_buffer: torch.Tensor, weights: Optional[torch.Tensor], regions: Sequence[tuple], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Everything after the custom regions' denoiser calls in one launch (multidiffusion.py:187-216,
    mixtureofdiffusers.py:145-175).  regions: [(x, y, w, h, mode, region_out [N,C,h,w], aux fp32 [h,w] or None)] in list
    order, mode 0 BACKGROUND (aux = optional multiplier) / 1 FOREGROUND (aux = feather mask).  weights: the fp32
    divide-where->1 canvas (MultiDiffusion) or None.  Returns fp32 [N,C,H,W]."""
    _require_cuda(x_buffer, "x_buffer")
    N, C, H, W = x_buffer.shape
    xb = x_buffer.contiguous()
    arr, keep = _region_table(xb, regions)
    res = out if out is not None else torch.empty((N, C, H, W), dtype=torch.float32, device=xb.device)
    with torch.cuda.device(xb.device):
        check(lib.td_region_composite(xb.data_ptr(), weights.data_ptr() if weights is not None else None, arr, len(regions), N, C, H, W,
                                      dtype_code(xb.dtype), res.data_ptr(), current_stream_ptr(xb.device)))
    return res


def region_composite_rows(x_buffer: torch.Tensor, weights: Optional[torch.Tensor], regions: Sequence[tuple], row_begin: int, row_end: int,
                          out: torch.Tensor) -> torch.Tensor:
    """`region_composite` of the canvas rows [row_begin, row_end) only, written into those rows of `out` (fp32 [N,C,H,W], the
    other rows are left as they are).  Regions are in canvas coordinates; one that is given clipped to the window (y, h and
    its output / aux narrowed to the rows it covers there) composites the same values."""
    _require_cuda(x_buffer, "x_buffer")
    N, C, H, W = x_buffer.shape
    if not x_buffer.is_contiguous() or not out.is_contiguous() or out.dtype != torch.float32 or tuple(out.shape) != (N, C, H, W):
        raise ValueError("region_composite_rows: x_buffer and out must be contiguous whole-canvas tensors, out fp32")
    arr, keep = _region_table(x_buffer, regions)
    with torch.cuda.device(x_buffer.device):
        check(lib.td_region_composite_rows(x_buffer.data_ptr(), weights.data_ptr() if weights is not None else None, arr, len(regions), N, C,
                                           H, W, dtype_code(x_buffer.dtype), out.data_ptr(), int(row_begin), int(row_end),
                                           current_stream_ptr(x_buffer.device)))
    return out
