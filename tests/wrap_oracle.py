"""Oracle for seamless (periodic) tiling: numpy / torch-CPU restatement of td_grid_init and td_grid_weights on a plan with
wrap bits, and of the scatter and both blends on such a plan.

Written from the plan's definition, with explicit per-tile loops and the same dtype round trips as oracle/blend.py:
the canvas accumulates in its dtype with one rounding per tile add in tile-list order, MultiDiffusion divides in fp32
where weights > 1, Mixture of Diffusers multiplies by the fp32 product tile_weights * rescale first.  A tile covers
canvas rows (y0 + v) mod H and columns (x0 + u) mod W on a wrapped axis.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

BBox = Tuple[int, int, int, int]  # x, y, w, h; x + w may exceed W on a wrapped axis

WRAP_X, WRAP_Y = 1, 2


def linear_origins(L: int, t: int, ov: int) -> List[int]:
    """split_bboxes' rule for one axis (tile_utils/utils.py:160-177)."""
    n = max(0, math.ceil((L - ov) / (t - ov)))
    d = (L - t) / (n - 1) if n > 1 else 0
    return [min(int(i * d), L - t) for i in range(n)]


def periodic_origins(L: int, t: int, ov: int) -> List[int]:
    """One tile at 0 when t == L, else n = ceil(L / (t - ov)) tiles at floor(k * L / n) (float64)."""
    if t == L:
        return [0]
    n = math.ceil(L / (t - ov))
    d = L / n
    return [math.floor(k * d) for k in range(n)]


class WrapPlan:
    """What init_grid_bbox(..., wrap_x, wrap_y) leaves on the delegate."""

    def __init__(self, w: int, h: int, tile_w: int, tile_h: int, overlap: int, tile_bs: int, wrap: int, gaussian: bool = False):
        from oracle import tiling
        self.w, self.h, self.wrap = w, h, wrap
        self.tile_w, self.tile_h = min(tile_w, w), min(tile_h, h)
        self.overlap = max(0, min(overlap, min(tile_w, tile_h) - 4))
        self.xs = (periodic_origins if wrap & WRAP_X else linear_origins)(w, self.tile_w, self.overlap)
        self.ys = (periodic_origins if wrap & WRAP_Y else linear_origins)(h, self.tile_h, self.overlap)
        self.bboxes = [(x, y, self.tile_w, self.tile_h) for y in self.ys for x in self.xs]
        n = len(self.bboxes)
        self.num_batches = math.ceil(n / tile_bs)
        self.tile_bs = math.ceil(n / self.num_batches)
        self.batched_bboxes = [self.bboxes[i * self.tile_bs:(i + 1) * self.tile_bs] for i in range(self.num_batches)]
        self.tile_weights = tiling.gaussian_weights(self.tile_w, self.tile_h) if gaussian else None
        self.weights = weights(self.bboxes, w, h, self.tile_weights)
        with np.errstate(divide="ignore"):
            self.rescale_factor = (np.float32(1.0) / self.weights).astype(np.float32)


def rows_cols(b: BBox, W: int, H: int):
    x, y, w, h = b
    return torch.arange(y, y + h) % H, torch.arange(x, x + w) % W


def weights(bboxes: Sequence[BBox], W: int, H: int, tile_weights: Optional[np.ndarray] = None) -> np.ndarray:
    """fp32 zeros, then `+= tile weight` per tile in list order at ((y + v) mod H, (x + u) mod W)."""
    out = np.zeros((H, W), dtype=np.float32)
    for (x, y, w, h) in bboxes:
        idx = (((y + np.arange(h)) % H)[:, None], ((x + np.arange(w)) % W)[None, :])   # distinct pixels within one tile
        add = np.ones((h, w), dtype=np.float32) if tile_weights is None else tile_weights
        out[idx] = out[idx] + add
    return out


def scatter(x: torch.Tensor, bboxes: Sequence[BBox]) -> torch.Tensor:
    """[N,C,H,W] -> [len(bboxes)*N, C, th, tw], tile-major, modular crop."""
    H, W = x.shape[2], x.shape[3]
    out = []
    for b in bboxes:
        iy, ix = rows_cols(b, W, H)
        out.append(x[:, :, iy][:, :, :, ix])
    return torch.cat(out, dim=0)


def accumulate_md(x_buffer: torch.Tensor, tile_out: torch.Tensor, bboxes: Sequence[BBox], N: int) -> None:
    H, W = x_buffer.shape[2], x_buffer.shape[3]
    for i, b in enumerate(bboxes):
        iy, ix = rows_cols(b, W, H)
        idx = (slice(None), slice(None), iy[:, None], ix[None, :])
        x_buffer[idx] = (x_buffer[idx] + tile_out[i * N:(i + 1) * N]).to(x_buffer.dtype)   # one rounding in the buffer dtype


def accumulate_mod(x_buffer: torch.Tensor, tile_out: torch.Tensor, bboxes: Sequence[BBox], N: int, tile_weights: torch.Tensor,
                   rescale: torch.Tensor) -> None:
    H, W = x_buffer.shape[2], x_buffer.shape[3]
    for i, b in enumerate(bboxes):
        iy, ix = rows_cols(b, W, H)
        idx = (slice(None), slice(None), iy[:, None], ix[None, :])
        wgt = tile_weights * rescale[idx]                                    # fp32 product
        x_buffer[idx] = (x_buffer[idx] + tile_out[i * N:(i + 1) * N] * wgt).to(x_buffer.dtype)


def normalise_md(x_buffer: torch.Tensor, weights_t: torch.Tensor) -> torch.Tensor:
    return torch.where(weights_t > 1, x_buffer / weights_t, x_buffer)


def blend_md(outs: Sequence[torch.Tensor], batched_bboxes, N: int, shape, dtype, weights_np: np.ndarray):
    """(fp32 normalised canvas, un-normalised accumulator in `dtype`)."""
    xb = torch.zeros(shape, dtype=dtype)
    for out, bbs in zip(outs, batched_bboxes):
        accumulate_md(xb, out.cpu(), bbs, N)
    w = torch.from_numpy(weights_np).view(1, 1, *weights_np.shape)
    return normalise_md(xb, w).float(), xb


def blend_mod(outs: Sequence[torch.Tensor], batched_bboxes, N: int, shape, dtype, tile_weights: np.ndarray, rescale: np.ndarray):
    xb = torch.zeros(shape, dtype=dtype)
    tw = torch.from_numpy(tile_weights)
    rs = torch.from_numpy(rescale).view(1, 1, *rescale.shape)
    for out, bbs in zip(outs, batched_bboxes):
        accumulate_mod(xb, out.cpu(), bbs, N, tw, rs)
    return xb


def multidiffusion_step(x: torch.Tensor, plan: WrapPlan, denoise: Callable[[torch.Tensor, Sequence[BBox]], torch.Tensor]):
    N = x.shape[0]
    outs = [denoise(scatter(x, bbs), bbs) for bbs in plan.batched_bboxes]
    return blend_md(outs, plan.batched_bboxes, N, x.shape, x.dtype, plan.weights)


def mixture_step(x: torch.Tensor, plan: WrapPlan, denoise: Callable[[torch.Tensor, Sequence[BBox]], torch.Tensor]):
    N = x.shape[0]
    outs = [denoise(scatter(x, bbs), bbs) for bbs in plan.batched_bboxes]
    return blend_mod(outs, plan.batched_bboxes, N, x.shape, x.dtype, plan.tile_weights, plan.rescale_factor)


def blur_denoise(x_tile: torch.Tensor, bboxes=None) -> torch.Tensor:
    """Tile-local stand-in for the UNet: a zero-padded 3x3 box blur (sum of the 9 neighbours / 16) in fp32, rounded
    to the tile dtype.  Every operation is an IEEE add or an exact power-of-two scale, so CPU and GPU agree bit for bit;
    a tile sees only its own pixels, like a UNet with zero padding."""
    f = torch.nn.functional.pad(x_tile.float(), (1, 1, 1, 1))
    h = f[:, :, :, :-2] + f[:, :, :, 1:-1]
    h = h + f[:, :, :, 2:]
    v = h[:, :, :-2] + h[:, :, 1:-1]
    v = v + h[:, :, 2:]
    return (v * 0.0625).to(x_tile.dtype)


# ------------------------------------------------------------------------------------------------ tiled VAE
def vae_split_wrap(h: int, w: int, tile_size: int, pad: int, is_decoder: bool, wrap: int):
    """td_vae_split_tiles with wrap bits: (in_bboxes, out_bboxes), [x1, x2, y1, y2] each, rows outer.  A non-wrapped axis is taken
    from oracle/vae.py's split_tiles; a wrapped axis of length L is cut at b_k = m * floor(k * L / (n * m)),
    n = max(ceil(L / tile), 1), b_n = L, input [b_k - pad, b_{k+1} + pad) unclipped."""
    from oracle import vae as ovae
    ib, ob = ovae.split_tiles(h, w, tile_size, pad, is_decoder)
    ncols = sum(1 for b in ib if b[2:] == ib[0][2:])
    bx = [(ib[j][0], ib[j][1], ob[j][0], ob[j][1]) for j in range(ncols)]
    by = [(ib[i * ncols][2], ib[i * ncols][3], ob[i * ncols][2], ob[i * ncols][3]) for i in range(len(ib) // ncols)]
    sc = (lambda v: v * 8) if is_decoder else (lambda v: v // 8)

    def periodic(L):
        m = 1 if is_decoder else 8
        n = max(math.ceil(L / tile_size), 1)
        cut = [m * ((k * L) // (n * m)) for k in range(n)] + [L]
        return [(cut[k] - pad, cut[k + 1] + pad, sc(cut[k]), sc(cut[k + 1])) for k in range(n)]

    if wrap & WRAP_X:
        bx = periodic(w)
    if wrap & WRAP_Y:
        by = periodic(h)
    in_b = [[x[0], x[1], y[0], y[1]] for y in by for x in bx]
    out_b = [[x[2], x[3], y[2], y[3]] for y in by for x in bx]
    return in_b, out_b


def load_wrap(z: torch.Tensor, b) -> torch.Tensor:
    """Tile [x1, x2) x [y1, y2) of a periodic canvas, bounds in unwrapped coordinates."""
    H, W = z.shape[2], z.shape[3]
    iy = torch.arange(b[2], b[3], device=z.device) % H
    ix = torch.arange(b[0], b[1], device=z.device) % W
    return z[:, :, iy][:, :, :, ix].clone()


def vae_tile_forward_wrap(net, z: torch.Tensor, tile_size: int, is_decoder: bool, fast_mode: bool, wrap: int,
                          color_fix: bool = False) -> torch.Tensor:
    """oracle/vae.py's vae_tile_forward on the periodic split: the same task queues, zig-zag rounds, merged GroupNorm
    statistics and fast-mode estimate (on the whole latent, as before); only the tile load reads modulo the canvas.  No
    tiny-input bypass: a wrapped seam always gets its halo."""
    from oracle import vae as ovae
    dtype = next(net.parameters()).dtype
    pad = 11 if is_decoder else 32
    color_fix = color_fix and not is_decoder
    z = z.detach()
    N, height, width = z.shape[0], z.shape[2], z.shape[3]
    in_bboxes, out_bboxes = vae_split_wrap(height, width, tile_size, pad, is_decoder, wrap)
    tiles = [load_wrap(z, b) for b in in_bboxes]
    T = len(tiles)
    ops = ovae.build_task_queue(net, is_decoder)
    if fast_mode:
        est_ops = ovae._clone_ops(ops)
        if ovae.estimate_group_norm(ovae.fast_mode_estimator_input(z, tile_size), est_ops, color_fix):
            ops = est_ops
    queues = [ovae._clone_ops(ops) for _ in range(T)]
    result = None
    done = 0
    forward = True
    while True:
        stats = ([], [], [])
        layer = None
        order = range(T) if forward else reversed(range(T))
        for i in order:
            tile, q = tiles[i], queues[i]
            while q:
                kind, fn = q.pop(0)
                if kind == "pre_norm":
                    var, mean = ovae.get_var_mean(tile)
                    stats[0].append(var); stats[1].append(mean); stats[2].append(tile.shape[2] * tile.shape[3])
                    layer = fn
                    break
                elif kind in ("store_res", "store_res_cpu"):
                    j = 0
                    while q[j][0] != "add_res":
                        j += 1
                    q[j][1] = fn(tile)
                elif kind == "add_res":
                    tile = tile + fn
                else:
                    tile = fn(tile)
            if not q:
                tiles[i] = None
                done += 1
                if result is None:
                    result = torch.zeros((N, tile.shape[1], height * 8 if is_decoder else height // 8,
                                          width * 8 if is_decoder else width // 8), dtype=torch.float32, device=z.device)
                ob = out_bboxes[i]
                result[:, :, ob[2]:ob[3], ob[0]:ob[1]] = ovae.crop_valid_region(tile, in_bboxes[i], ob, is_decoder)
            else:
                tiles[i] = tile
                if i == T - 1 and forward:
                    forward = False
                elif i == 0 and not forward:
                    forward = True
        if done == T:
            break
        if stats[0]:
            var, mean = ovae.merge_tile_stats(*stats)
            weight, bias = getattr(layer, "weight", None), getattr(layer, "bias", None)
            norm = lambda x, mean=mean, var=var, weight=weight, bias=bias: ovae.custom_group_norm(x, mean, var, weight, bias)
            for q in queues:
                if q:
                    q.insert(0, ["apply_norm", norm])
    return result.to(dtype)
