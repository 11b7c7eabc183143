"""SpotDiffusion (Frolov et al., 2024) tile method: MultiDiffusion's blend on sparse windows that move on every denoiser call.

New: the reference has no such method.  The windows barely overlap, so a call costs far fewer UNet evaluations than
MultiDiffusion at its default overlap; a seam left by one call lies inside a window at the next call and is denoised there.
Each tiled denoiser call runs

    shift draw (random.Random(shift_seed), x then y)
    td_grid_shift             the step plan: the base plan's windows moved back by the shift (host, O(tiles))
    td_grid_counts            its count canvas and exact reciprocals, written on the device into persistent buffers
    td_scatter_tiles          -> UNet batches ->  td_blend_multidiffusion   (as MultiDiffusion, on the step plan)

so no weight canvas is built on the host or uploaded per call.  The step plans are defined in include/td_b200.h.
"""
from __future__ import annotations

import random
from typing import Callable, Optional

import torch
from torch import Tensor

from .. import engine
from ..host import opt_f
from ..tile_utils.utils import grid_bbox
from .multidiffusion import MultiDiffusion


class SpotDiffusion(MultiDiffusion):

    def __init__(self, p, *args, **kwargs):
        super().__init__(p, *args, **kwargs)
        self._base_grid = None                  # td_grid_init plan the step plans are shifted from
        self._shift_bounds = None               # (lo_x, hi_x, lo_y, hi_y)
        self._shift_rng: Optional[random.Random] = None
        self._tile_bs_arg: Optional[int] = None
        self._rcp_buf: Optional[Tensor] = None  # persistent RN(1/weights) canvas; `weights` is the count canvas

    @grid_bbox
    def init_grid_bbox(self, tile_w: int, tile_h: int, overlap: int, tile_bs: int, wrap_x: bool = False, wrap_y: bool = False,
                       shift_seed: int = 0):
        """The base plan is MultiDiffusion's (td_grid_init: clamps, overlap rule, periodic axes); every tiled denoiser call
        then draws a shift and runs on the step plan (td_grid_shift).  The window count does not depend on the shift, so
        num_tiles / num_batches / tile_bs are fixed for the job; `batched_bboxes` is the current call's list."""
        wrap = (engine.WRAP_X if wrap_x else 0) | (engine.WRAP_Y if wrap_y else 0)
        base = engine.make_grid(self.w, self.h, tile_w, tile_h, overlap, tile_bs, wrap=wrap)
        bounds = engine.shift_bounds(base)
        first = engine.shift_grid(base, bounds[0], bounds[2], tile_bs)     # refuses a plan that cannot grow before any state changes
        self.enable_grid_bbox = True
        self._base_grid, self._shift_bounds, self._tile_bs_arg = base, bounds, int(tile_bs)
        self._shift_rng = random.Random(shift_seed)
        self.tile_w, self.tile_h = int(base.tile_w), int(base.tile_h)
        self._grid = first
        self._set_grid_bboxes(first)

    def _init_rcp_weights(self):
        self._rcp_weights = None            # written with the count canvas by every call

    # ------------------------------------------------------------- refused
    def init_custom_bbox(self, *args, **kwargs):
        raise NotImplementedError("SpotDiffusion does not support region prompt control")

    def init_tile_shard(self, *args, **kwargs):
        raise NotImplementedError("SpotDiffusion does not support the multi-GPU tile shard")

    def init_noise_inverse(self, *args, **kwargs):
        raise NotImplementedError("SpotDiffusion does not support noise inversion")

    def init_inpaint_mask(self, *args, **kwargs):
        raise NotImplementedError("SpotDiffusion does not support the inpaint mask: its windows move every step")

    # ------------------------------------------------------------- per call
    def draw_shift(self):
        """(shift_x, shift_y) of the next call: randrange(lo, hi) for x, then for y; an axis with one allowed shift draws nothing."""
        lo_x, hi_x, lo_y, hi_y = self._shift_bounds
        sx = self._shift_rng.randrange(lo_x, hi_x) if hi_x - lo_x > 1 else lo_x
        sy = self._shift_rng.randrange(lo_y, hi_y) if hi_y - lo_y > 1 else lo_y
        return sx, sy

    def _next_plan(self, device: torch.device):
        sx, sy = self.draw_shift()
        g = engine.shift_grid(self._base_grid, sx, sy, self._tile_bs_arg)
        self._grid = g
        self._set_grid_bboxes(g)
        fast = engine.counts_allow_fast_divide(g)
        if fast and (self._rcp_buf is None or self._rcp_buf.device != device):
            self._rcp_buf = torch.empty((self.h, self.w), dtype=torch.float32, device=device)
        engine.grid_counts(g, self.weights, self._rcp_buf if fast else None)
        self._rcp_weights = self._rcp_buf if fast else None
        # side inputs are cropped with the plan of this call (the per-job crops of the base class would not match the tiles)
        if self._control_params():
            self.control_tensor_batch = [self._side_input_tiles(hint, opt_f, self.control_tensor_cpu)[0]
                                         for hint in self.org_control_tensor_batch]
        if self._stablesr_model() is not None and self.stablesr_tensor is not None:
            self.stablesr_tensor_batch = self._side_input_tiles(self.stablesr_tensor, 1, False)[0]

    def sample_one_step(self, x_in: Tensor, org_func: Callable, repeat_func: Callable, custom_func: Callable) -> Tensor:
        """MultiDiffusion's step on a fresh step plan.  The hires-fix second pass (another latent size) is not tiled and draws
        no shift."""
        if self.enable_grid_bbox and tuple(x_in.shape[2:]) == (self.h, self.w):
            x = self._check_input(x_in)         # weights follow the latent's device
            self._next_plan(x.device)
        return super().sample_one_step(x_in, org_func, repeat_func, custom_func)
