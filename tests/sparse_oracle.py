"""Oracle for the sparse blends (td_blend_multidiffusion_sparse / td_blend_mixture_sparse), and a CPU model of their
cp.async visit tables for the injected-defect checks.

A sparse blend is the dense blend of the full plan with the skipped tiles left out: oracle/blend.py's accumulation over
the kept tiles only, in tile order, with the full plan's weights (MultiDiffusion) or tile weights and rescale factor
(Mixture of Diffusers).  Nothing here reads a device kernel, so the expected bits -- signed zeros included -- do not
depend on the dense CUDA blend being right.

`emulate` restates how the cp.async kernels walk a patch: the tiles touching an 8-row x 8-vector patch, in ascending
tile order, compacted to the kept ones (prepare_sparse_visits), then consumed visit by visit.  Without a defect it
gives the oracle's bits; each defect breaks the table of one patch the way a faulty compaction would.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from oracle import blend

BBox = Tuple[int, int, int, int]
PATCH_ROWS, PATCH_VECS = 8, 8           # kAsY, kAsX of csrc/td_diffusion.cu


def _kept(tiles: torch.Tensor, bboxes: Sequence[BBox], active: np.ndarray, N: int):
    idx = [t for t in range(len(bboxes)) if active[t]]
    if not idx:
        return None, []
    rows = torch.tensor([t * N + n for t in idx for n in range(N)], dtype=torch.long)
    return tiles.index_select(0, rows), [bboxes[t] for t in idx]


def sparse_md(tiles: torch.Tensor, bboxes: Sequence[BBox], active: np.ndarray, N: int, weights: np.ndarray,
              acc_dtype: torch.dtype):
    """(x_out fp32, x_buffer in acc_dtype): tiles [T*N, C, th, tw] are the full plan's outputs in tile order; only those
    with active[t] are added."""
    T = len(bboxes)
    assert tiles.shape[0] == T * N
    H, W = weights.shape
    buf = torch.zeros((N, tiles.shape[1], H, W), dtype=acc_dtype)
    kept, kb = _kept(tiles, bboxes, active, N)
    if kb:
        blend.accumulate_md(buf, kept, kb, N)
    return blend.normalise_md(buf, torch.from_numpy(weights).view(1, 1, H, W)).float(), buf


def sparse_mod(tiles: torch.Tensor, bboxes: Sequence[BBox], active: np.ndarray, N: int, tile_weights: np.ndarray,
               rescale: np.ndarray, acc_dtype: torch.dtype) -> torch.Tensor:
    """x_buffer in acc_dtype (Mixture of Diffusers' result is the buffer)."""
    H, W = rescale.shape
    buf = torch.zeros((N, tiles.shape[1], H, W), dtype=acc_dtype)
    kept, kb = _kept(tiles, bboxes, active, N)
    if kb:
        blend.accumulate_mod(buf, kept, kb, N, torch.from_numpy(tile_weights), torch.from_numpy(rescale).view(1, 1, H, W))
    return buf


def patch_tables(xs: Sequence[int], ys: Sequence[int], tw: int, th: int, W: int, H: int, es: int):
    """[((x0, y0, x1, y1), [tile indices in table order])] of every cp.async patch (fill_patch_table: the tile rows and
    columns touching the patch, row-major, i.e. ascending tile order)."""
    bx = PATCH_VECS * (16 // es)
    out = []
    for y0 in range(0, H, PATCH_ROWS):
        y1 = min(y0 + PATCH_ROWS, H)
        rs = [r for r, y in enumerate(ys) if y < y1 and y + th > y0]
        for x0 in range(0, W, bx):
            x1 = min(x0 + bx, W)
            cs = [c for c, x in enumerate(xs) if x < x1 and x + tw > x0]
            out.append(((x0, y0, x1, y1), [r * len(xs) + c for r in rs for c in cs]))
    return out


def kept_table(table: Sequence[int], active: np.ndarray):
    return [t for t in table if active[t]]


def fullest_patch(tables, active: Optional[np.ndarray] = None):
    """Index of the patch holding the most (kept) visits."""
    counts = [len(t if active is None else kept_table(t, active)) for _, t in tables]
    return int(np.argmax(counts))


def emulate(mode: str, tiles: torch.Tensor, xs, ys, tw: int, th: int, active: np.ndarray, N: int, acc_dtype: torch.dtype,
            es: int, weights: Optional[np.ndarray] = None, tile_weights: Optional[np.ndarray] = None,
            rescale: Optional[np.ndarray] = None, defect: Optional[tuple] = None):
    """The sparse cp.async blend patch by patch.  `defect` = (kind, patch, *args) alters that patch's kept-visit table:
    ("drop", p, i) loses position i, ("swap", p, i, j) exchanges positions i and j, ("include", p, t) adds skipped tile t
    at its place in tile order (read from `tiles`, which holds every tile's output).  Returns what sparse_md / sparse_mod
    return."""
    H, W = (weights if weights is not None else rescale).shape
    C = tiles.shape[1]
    buf = torch.zeros((N, C, H, W), dtype=acc_dtype)
    tables = patch_tables(xs, ys, tw, th, W, H, es)
    cols = len(xs)
    tw_t = torch.from_numpy(tile_weights) if tile_weights is not None else None
    rs_t = torch.from_numpy(rescale).view(1, 1, H, W) if rescale is not None else None
    for p, ((x0, y0, x1, y1), table) in enumerate(tables):
        visits = kept_table(table, active)
        if defect is not None and defect[1] == p:
            kind = defect[0]
            if kind == "drop":
                del visits[defect[2]]
            elif kind == "swap":
                i, j = defect[2], defect[3]
                visits[i], visits[j] = visits[j], visits[i]
            elif kind == "include":
                assert not active[defect[2]] and defect[2] in table
                visits = sorted(visits + [defect[2]])
        for t in visits:
            tx, ty = xs[t % cols], ys[t // cols]
            a0, a1, b0, b1 = max(x0, tx), min(x1, tx + tw), max(y0, ty), min(y1, ty + th)
            if a0 >= a1 or b0 >= b1:
                continue
            src = tiles[t * N:(t + 1) * N, :, b0 - ty:b1 - ty, a0 - tx:a1 - tx]
            dst = buf[:, :, b0:b1, a0:a1]
            if mode == "md":
                dst += src
            else:
                dst += src * (tw_t[b0 - ty:b1 - ty, a0 - tx:a1 - tx] * rs_t[:, :, b0:b1, a0:a1])
    if mode == "md":
        return blend.normalise_md(buf, torch.from_numpy(weights).view(1, 1, H, W)).float(), buf
    return buf
