"""Oracle for SpotDiffusion: a restatement of the step plan (include/td_b200.h, td_grid_shift) with explicit per-axis loops,
of the shift schedule, and of one step.

The step is MultiDiffusion's blend on the step plan's window list: oracle/blend.py's op sequence on a bounded canvas and
tests/wrap_oracle.py's modular one when an axis is wrapped (adds in tile order rounded to the latent dtype, then
where(count > 1, acc / count, acc) in fp32).
"""
from __future__ import annotations

import math
import random
from typing import Callable, List, Sequence, Tuple

import numpy as np
import torch

import wrap_oracle as wo
from oracle import blend

WRAP_X, WRAP_Y = wo.WRAP_X, wo.WRAP_Y


def base_axis(L: int, t: int, ov: int, periodic: bool) -> List[int]:
    return (wo.periodic_origins if periodic else wo.linear_origins)(L, t, ov)


def smallest_gap(b: Sequence[int], L: int, periodic: bool) -> int:
    n = len(b)
    if n == 1:
        return L
    gap = None
    for k in range(1, n):
        d = b[k] - b[k - 1]
        gap = d if gap is None else min(gap, d)
    if periodic:
        gap = min(gap, L + b[0] - b[n - 1])
    return gap


def shift_range(b: Sequence[int], L: int, periodic: bool) -> Tuple[int, int]:
    """[lo, hi) of the shifts one axis accepts."""
    g = smallest_gap(b, L, periodic)
    if periodic:
        return 0, g
    if len(b) >= 2 and g >= 2:
        return 1, g
    return 0, 1


def step_axis(b: Sequence[int], L: int, t: int, periodic: bool, s: int) -> List[int]:
    lo, hi = shift_range(b, L, periodic)
    assert lo <= s < hi, (s, lo, hi)
    if periodic:
        out = []
        for o in b:
            out.append((o - s) % L)
        return sorted(out)
    if lo == 0:
        return list(b)
    out = [0]
    for k in range(1, len(b)):
        out.append(b[k] - s)
    out.append(L - t)
    return out


def coverage(origins: Sequence[int], L: int, t: int, periodic: bool) -> np.ndarray:
    """Windows covering each position of an axis, counted window by window."""
    out = np.zeros(L, dtype=np.int64)
    for o in origins:
        for u in range(t):
            p = o + u
            if periodic:
                p %= L
            out[p] += 1
    return out


class SpotPlan:
    """The step plan of (shift_x, shift_y), with the attributes wrap_oracle's step reads."""

    def __init__(self, w: int, h: int, tile_w: int, tile_h: int, overlap: int, tile_bs: int, wrap: int, shift_x: int, shift_y: int):
        self.w, self.h, self.wrap = w, h, wrap
        self.tile_w, self.tile_h = min(tile_w, w), min(tile_h, h)
        self.overlap = max(0, min(overlap, min(tile_w, tile_h) - 4))
        px, py = bool(wrap & WRAP_X), bool(wrap & WRAP_Y)
        self.base_xs = base_axis(w, self.tile_w, self.overlap, px)
        self.base_ys = base_axis(h, self.tile_h, self.overlap, py)
        self.xs = step_axis(self.base_xs, w, self.tile_w, px, shift_x)
        self.ys = step_axis(self.base_ys, h, self.tile_h, py, shift_y)
        self.bboxes = [(x, y, self.tile_w, self.tile_h) for y in self.ys for x in self.xs]
        n = len(self.bboxes)
        self.num_batches = math.ceil(n / tile_bs)
        self.tile_bs = math.ceil(n / self.num_batches)
        self.batched_bboxes = [self.bboxes[i * self.tile_bs:(i + 1) * self.tile_bs] for i in range(self.num_batches)]
        self.weights = wo.weights(self.bboxes, w, h)


def bounds(w: int, h: int, tile_w: int, tile_h: int, overlap: int, wrap: int) -> Tuple[int, int, int, int]:
    tw, th = min(tile_w, w), min(tile_h, h)
    ov = max(0, min(overlap, min(tile_w, tile_h) - 4))
    px, py = bool(wrap & WRAP_X), bool(wrap & WRAP_Y)
    return shift_range(base_axis(w, tw, ov, px), w, px) + shift_range(base_axis(h, th, ov, py), h, py)


def schedule(seed: int, rng_bounds: Tuple[int, int, int, int], calls: int) -> List[Tuple[int, int]]:
    """The shifts of `calls` consecutive tiled calls: randrange for x, then for y, nothing on a single-value axis."""
    rng = random.Random(seed)
    lo_x, hi_x, lo_y, hi_y = rng_bounds
    out = []
    for _ in range(calls):
        sx = rng.randrange(lo_x, hi_x) if hi_x - lo_x > 1 else lo_x
        sy = rng.randrange(lo_y, hi_y) if hi_y - lo_y > 1 else lo_y
        out.append((sx, sy))
    return out


def step(x: torch.Tensor, plan: SpotPlan, denoise: Callable[[torch.Tensor, Sequence], torch.Tensor]) -> torch.Tensor:
    """One SpotDiffusion denoiser call: fp32 [N,C,H,W]."""
    if plan.wrap:
        return wo.multidiffusion_step(x, plan, denoise)[0]
    return blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, denoise).float()
