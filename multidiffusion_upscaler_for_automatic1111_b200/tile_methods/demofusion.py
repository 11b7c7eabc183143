"""DemoFusion (arXiv 2311.16973) tile method with the reference's surface
(tile_methods/demofusion.py), on the sm_90a kernels:

    local windows   td_scatter_tiles + td_blend_multidiffusion (count-normalised)     demofusion.py:254-264
    gaussian blur   td_depthwise_conv2d                                                demofusion.py:173-178
    renormalise     td_gn_stats (whole-tensor mean / unbiased std) + td_affine_clamp   demofusion.py:269-273
    global views    td_dilated_gather                                                  demofusion.py:283-308
    add-back + mix  td_demofusion_combine (one launch)                                 demofusion.py:296-322

Random jitter (demofusion.py:116-134, offsets from Python's `random`) makes the window list non-separable: the
local windows then go through the list-driven td_scatter_bboxes / td_blend_bboxes on the zero-padded latent and the
add-back through td_demofusion_combine_offset (csrc/td_jitter.cu).

Seamless tiling (new: the reference has no periodic canvas), get_views(..., wrap_x, wrap_y): the local windows are the
periodic plan of td_grid_init (ring windows, count-normalised through td_wrap.cu), or with random jitter a ring window list
on td_scatter_bboxes_wrap / td_blend_bboxes_wrap; the gaussian filter indexes the wrapped axes circularly
(td_depthwise_conv2d_wrap).  The latent is never padded then: a jittered window on a bounded axis reads zeros off the
canvas and drops them in the blend, and the dilated views cover the whole canvas from 0.  tests/demofusion_wrap_oracle.py
(demofusion_views, demofusion_step) defines these semantics.
"""
from __future__ import annotations

import ctypes
import math
import random
from typing import Dict, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from .. import engine, host, tilevae
from .._cabi import check, current_stream_ptr, dtype_code, lib
from ..tile_utils.utils import BBox, grid_bbox, keep_signature
from .abstractdiffusion import AbstractDiffusion, CondDict


class DemoFusion(AbstractDiffusion):

    def __init__(self, p, *args, **kwargs):
        super().__init__(p, *args, **kwargs)
        assert p.sampler_name != 'UniPC', 'Demofusion is not compatible with UniPC!'
        self.jitter_range = 0
        self.repeat_3 = False
        self._jitter = False                 # window LIST (random jitter) instead of the separable grid
        self._wrap = 0                       # engine.WRAP_X | WRAP_Y: periodic canvas axes (get_views' wrap_x / wrap_y)
        self._origins_host = None
        self._origins_dev = None
        self._shard_on = False               # tile shard requested (init_tile_shard); re-derived by every get_views
        self._view_shard = None

    @property
    def _list_wrap(self) -> dict:
        """The window-list engine calls take `wrap` only on a seamless canvas (the bounded calls are unchanged)."""
        return {"wrap": self._wrap} if self._wrap else {}

    def _check_input(self, x_in: Tensor) -> Tensor:
        if not self._jitter:
            return super()._check_input(x_in)
        if not x_in.is_cuda:
            raise RuntimeError(f"{self.method}: latent is on {x_in.device}; the H100 path has no CPU fallback")
        if self._origins_dev is None:
            raise RuntimeError(f"{self.method}: get_views() has not been called")
        return x_in.contiguous()

    # ------------------------------------------------------------------ hooks
    def hook(self):
        """demofusion.py:21-35: replaces CFGDenoiser.forward; inner_model.forward is patched per call."""
        steps_fn = getattr(host._a1111("sd_samplers_common"), "setup_img2img_steps", None) if host._a1111("sd_samplers_common") else None
        steps = getattr(self.p, "steps", None)
        if steps_fn is not None:
            steps, self.t_enc = steps_fn(self.p, None)      # with opts.img2img_fix_steps the returned steps differ from p.steps
        else:
            self.t_enc = getattr(self.p, "t_enc", getattr(self.p, "steps", 1) - 1)
        cfg = self.sampler.model_wrap_cfg
        cfg.forward_ori = cfg.forward
        self.sampler_forward = cfg.inner_model.forward
        cfg.forward = self.forward_one_step
        if not self.is_kdiff:
            self.timesteps = self.sampler.get_timesteps(self.p, steps)     # demofusion.py:22,35: the steps setup_img2img_steps returned

    @staticmethod
    def unhook():
        sd_model = getattr(host.get_shared(), "sd_model", None)
        if sd_model is not None and hasattr(sd_model, 'apply_model_ori'):
            sd_model.apply_model = sd_model.apply_model_ori
            del sd_model.apply_model_ori

    # ------------------------------------------------------------------ views
    def global_split_bboxes(self) -> List[Tuple[int, int]]:
        """demofusion.py:87-99: the s*s dilated views (x, y), doubled in mixture mode."""
        s = self.p.current_scale_num
        views = [(col, row) for row in range(s) for col in range(s)]
        return views + views if self.p.mixture else views

    def split_bboxes_jitter(self, w_l: int, h_l: int, tile_w: int, tile_h: int, overlap: int = 16) -> List[BBox]:
        """demofusion.py:101-139 with random_jitter on: the regular window grid, every window moved by a random offset
        of at most jitter_range towards the inside (border windows only inwards), in coordinates of the latent
        zero-padded by jitter_range.  Offsets come from Python's global `random`, x before y, row-major -- the same
        draws as the reference, so a seeded run reproduces its windows."""
        cols = math.ceil((w_l - overlap) / (tile_w - overlap)) or 1
        rows = math.ceil((h_l - overlap) / (tile_h - overlap)) or 1
        dx = (w_l - tile_w) / (cols - 1) if cols > 1 else 0
        dy = (h_l - tile_h) / (rows - 1) if rows > 1 else 0
        jr = min(max((min(self.w, self.h) - self.stride) // 4, 0), min(int(self.window_size / 2), int(self.overlap / 2)))
        self.jitter_range = jr

        def draw(pos: int, size: int, extent: int) -> int:
            at_start, at_end = pos == 0, pos + size == extent
            if not at_start and not at_end:
                return random.randint(-jr, jr)
            if at_start and not at_end:
                return random.randint(-jr, 0)
            if at_end and not at_start:
                return random.randint(0, jr)
            return 0
        out = []
        for row in range(rows):
            for col in range(cols):
                y = min(int(row * dy), h_l - tile_h)
                x = min(int(col * dx), w_l - tile_w)
                xj = draw(x, tile_w, w_l)
                yj = draw(y, tile_h, h_l)
                out.append(BBox(x + xj + jr, y + yj + jr, tile_w, tile_h))
        return out

    def split_bboxes_jitter_wrap(self, g) -> List[BBox]:
        """Random jitter on the periodic plan `g` (seamless tiling): the windows of the plan in row-major order, each moved
        by draws from Python's global `random`, x before y, with the reference's jitter_range.  On a wrapped axis every
        window draws randint(-jr, jr) and its origin is kept mod L; on a bounded axis the reference's border rule holds
        (split_bboxes_jitter) and the origin is in canvas coordinates (no padding: it may start at -jr or end jr past L)."""
        jr = min(max((min(self.w, self.h) - self.stride) // 4, 0), min(int(self.window_size / 2), int(self.overlap / 2)))
        self.jitter_range = jr
        ws = self.window_size

        def draw(pos: int, size: int, extent: int, wrapped: bool) -> int:
            at_start, at_end = pos == 0, pos + size == extent
            if wrapped or (not at_start and not at_end):
                return random.randint(-jr, jr)
            if at_start and not at_end:
                return random.randint(-jr, 0)
            if at_end and not at_start:
                return random.randint(0, jr)
            return 0
        wx, wy = bool(self._wrap & engine.WRAP_X), bool(self._wrap & engine.WRAP_Y)
        out = []
        for x, y, _, _ in engine.grid_bboxes_xywh(g):
            x, y = int(x), int(y)
            xj = draw(x, ws, self.w, wx)
            yj = draw(y, ws, self.h, wy)
            out.append(BBox((x + xj) % self.w if wx else x + xj, (y + yj) % self.h if wy else y + yj, ws, ws))
        return out

    @grid_bbox
    def get_views(self, overlap: int, tile_bs: int, tile_bs_g: int, wrap_x: bool = False, wrap_y: bool = False):
        """demofusion.py:140-162: local window grid (stride = max(4, window - overlap)) + global view batches.

        wrap_x / wrap_y (the WebUI's "Tiling" option, passed again every upscaling phase) make the canvas periodic on that
        axis: seamless output.  The windows then run around the circle, and the latent is not padded for jitter."""
        self.enable_grid_bbox = True
        self.tile_w = self.tile_h = self.window_size
        self.overlap = max(0, min(overlap, self.window_size - 4))
        self.stride = max(4, self.window_size - self.overlap)
        self.jitter_range = 0
        self._jitter = bool(getattr(self.p, "random_jitter", False))
        self._wrap = (engine.WRAP_X if wrap_x else 0) | (engine.WRAP_Y if wrap_y else 0)
        if self._jitter:
            if self._wrap:
                g = engine.make_grid(self.w, self.h, self.window_size, self.window_size, self.overlap, tile_bs, wrap=self._wrap)
                if g.overlap != self.overlap or g.tile_w != self.window_size or g.tile_h != self.window_size:
                    raise ValueError("window larger than the latent: DemoFusion clamps window_size before get_views")
                bboxes = self.split_bboxes_jitter_wrap(g)
            else:
                bboxes = self.split_bboxes_jitter(self.w, self.h, self.tile_w, self.tile_h, self.overlap)
            self._grid = None
            flat = [v for b in bboxes for v in (b.x, b.y)]
            self._origins_host = (ctypes.c_int32 * len(flat))(*flat)
            self._origins_dev = torch.tensor(flat, dtype=torch.int32, device=host.device())
            self.num_tiles = len(bboxes)
            self.num_batches = math.ceil(self.num_tiles / tile_bs)
            self.tile_bs = math.ceil(self.num_tiles / self.num_batches)
        else:
            # split_bboxes_jitter without jitter is split_bboxes on the clamped overlap (demofusion.py:101-115);
            # init through td_grid_init with tile == window reproduces rows / cols / origins exactly
            g = engine.make_grid(self.w, self.h, self.window_size, self.window_size, self.overlap, tile_bs, wrap=self._wrap)
            if g.overlap != self.overlap or g.tile_w != self.window_size or g.tile_h != self.window_size:
                raise ValueError("window larger than the latent: DemoFusion clamps window_size before get_views")
            self._grid = g
            bboxes = [BBox(int(x), int(y), int(w), int(h)) for x, y, w, h in engine.grid_bboxes_xywh(g)]
            self.num_tiles = len(bboxes)
            self.num_batches = int(g.num_batches)
            self.tile_bs = int(g.tile_bs)
            counts = engine.grid_weights(g)   # how many windows cover each pixel (demofusion.py:261)
            counts[counts == 0] = 1.0         # :262
            self._counts = torch.from_numpy(counts).to(host.device())
            self._rcp_counts = torch.from_numpy(engine.exact_reciprocals(counts)).to(host.device())
        self.batched_bboxes = [bboxes[i * self.tile_bs:(i + 1) * self.tile_bs] for i in range(self.num_batches)]

        global_bboxes = self.global_split_bboxes()
        self.global_num_tiles = len(global_bboxes)
        self.global_num_batches = math.ceil(self.global_num_tiles / tile_bs_g)
        self.global_tile_bs = math.ceil(len(global_bboxes) / self.global_num_batches)
        self.global_batched_bboxes = [global_bboxes[i * self.global_tile_bs:(i + 1) * self.global_tile_bs]
                                      for i in range(self.global_num_batches)]
        if self._shard_on:
            self._derive_shards()

    def init_inpaint_mask(self, *args, **kwargs):
        raise NotImplementedError("DemoFusion does not support the inpaint mask: its global views cover the whole canvas")

    # ------------------------------------------------------------------ multi-GPU
    def init_tile_shard(self, group=None, fused: bool = False):
        """Shard the local windows AND the s*s global views over the ranks of `group` (one process per GPU): contiguous
        chunks of both lists; per step two all-gathers (window outputs, view outputs), then every rank runs the same
        ordered blend / add-back -- bit-identical across ranks and to a single-GPU run.  Survives get_views() (each
        upscaling phase rebuilds the lists).  With random jitter every rank must draw the same windows: seed Python's
        `random` identically on all ranks before get_views()."""
        if fused:
            raise NotImplementedError("DemoFusion shards through all-gather; the fused peer exchange is MultiDiffusion-only")
        self._shard_on, self._shard_group = True, group
        if self.batched_bboxes:
            self._derive_shards()
        return self._shard

    def _derive_shards(self):
        import torch.distributed as dist
        from .. import parallel
        rank, world = dist.get_rank(self._shard_group), dist.get_world_size(self._shard_group)
        self._shard = parallel.TileShard(self.num_tiles, rank, world)
        self._view_shard = parallel.TileShard(self.global_num_tiles, rank, world)
        windows = [b for batch in self.batched_bboxes for b in batch][self._shard.begin:self._shard.end]
        self.local_batched_bboxes = [windows[i:i + self.tile_bs] for i in range(0, len(windows), self.tile_bs)]
        views = [v for batch in self.global_batched_bboxes for v in batch][self._view_shard.begin:self._view_shard.end]
        self.local_global_batched_bboxes = [views[i:i + self.global_tile_bs] for i in range(0, len(views), self.global_tile_bs)]

    def _gather_chunks(self, outs, sh, rows_per_unit: int, unit_shape, dt, dev):
        """Pad this rank's outputs to the chunk size, all-gather, and return one tensor view per rank chunk (exact unit
        counts) -- the pointer-table form the blend / combine kernels take (`tile_bs` = chunk)."""
        from .. import parallel
        local = torch.zeros((sh.chunk * rows_per_unit,) + tuple(unit_shape), dtype=dt, device=dev)
        if outs:
            torch.cat(outs, dim=0, out=local[:sh.num_local * rows_per_unit])
        gathered = parallel.gather_tile_outputs(local, self._shard_group)
        chunks = []
        for b in range(sh.num_chunks):
            n = min(sh.chunk, sh.num_tiles - b * sh.chunk)
            chunks.append(gathered[b * sh.chunk * rows_per_unit:(b * sh.chunk + n) * rows_per_unit])
        return chunks

    def repeat_cond_dict(self, cond_in: CondDict, bboxes, mode) -> CondDict:
        """demofusion.py:60-84: text / vector cond repeated; spatial icond cropped (local) or dilated (global)."""
        n_rep = len(bboxes)
        tcond = self.repeat_tensor(self.get_tcond(cond_in), n_rep)
        icond = self.get_icond(cond_in)
        if tuple(icond.shape[2:]) == (self.h, self.w):
            if mode == 0 and self._wrap:  # ring windows: modular on the wrapped axes, zeros off a bounded one (as the latent)
                flat = [v for b in bboxes for v in (b.x, b.y)]
                origins_host = (ctypes.c_int32 * len(flat))(*flat)
                origins_dev = torch.tensor(flat, dtype=torch.int32, device=icond.device)
                icond = engine.scatter_bboxes(icond, origins_dev, origins_host, n_rep, self.window_size, self.window_size, wrap=self._wrap)
            elif mode == 0:
                if self._jitter:          # the windows live on the padded latent (demofusion.py:71-73)
                    jr = self.jitter_range
                    icond = F.pad(icond, (jr, jr, jr, jr), "constant", value=0)
                icond = torch.cat([icond[b.slicer] for b in bboxes], dim=0)
            else:
                s = self.p.current_scale_num
                icond = torch.cat([icond[:, :, b[1]::s, b[0]::s] for b in bboxes], dim=0)
        else:
            icond = self.repeat_tensor(icond, n_rep)
        vcond = self.get_vcond(cond_in)
        if vcond is not None:
            vcond = self.repeat_tensor(vcond, n_rep)
        return self.make_cond_dict(cond_in, tcond, icond, vcond)

    # ------------------------------------------------------------------ gaussian filter
    def gaussian_kernel(self, kernel_size=3, sigma=1.0, channels=3):
        """demofusion.py:164-171 (fp32, host)."""
        x_coord = torch.arange(kernel_size)
        g1 = torch.exp(-(x_coord - (kernel_size - 1) / 2) ** 2 / (2 * sigma ** 2))
        g1 = g1 / g1.sum()
        g2 = g1[:, None] * g1[None, :]
        return g2[None, None, :, :].repeat(channels, 1, 1, 1)

    def gaussian_filter(self, latents: Tensor, kernel_size=3, sigma=1.0) -> Tensor:
        """demofusion.py:173-178 as one depthwise stencil launch (weights rounded to the latent dtype like `.to(dtype)`);
        circular on the wrapped axes of a seamless canvas (td_depthwise_conv2d_wrap)."""
        k2 = self.gaussian_kernel(kernel_size, sigma, 1)[0, 0].to(latents.dtype).float().contiguous().numpy()
        x = latents.contiguous()
        out = torch.empty_like(x)
        n, c, hh, ww = x.shape
        with torch.cuda.device(x.device):
            if self._wrap:
                check(lib.td_depthwise_conv2d_wrap(x.data_ptr(), out.data_ptr(), n * c, hh, ww, k2.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                                   int(kernel_size), self._wrap, dtype_code(x.dtype), current_stream_ptr(x.device)))
            else:
                check(lib.td_depthwise_conv2d(x.data_ptr(), out.data_ptr(), n * c, hh, ww, k2.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                              int(kernel_size), dtype_code(x.dtype), current_stream_ptr(x.device)))
        return out

    def _renormalise(self, g_: Tensor, x_in: Tensor) -> Tensor:
        """(g - g.mean()) / g.std() * x.std() + x.mean() (demofusion.py:269,273), statistics in fp32, ops rounded in dtype."""
        dev = x_in.device

        def mean_std(t):
            var, mean = tilevae._segment_stats(t.contiguous(), 1, t.numel(), unbiased=True)
            return mean.to(t.dtype).float(), var.sqrt().to(t.dtype).float()   # the reference's 0-dim stats are dtype tensors
        mean_g, std_g = mean_std(g_)
        mean_x, std_x = mean_std(x_in)
        lo = torch.full((1,), -float("inf"), device=dev)
        hi = torch.full((1,), float("inf"), device=dev)
        n, c, hh, ww = g_.shape
        with torch.cuda.device(dev):
            check(lib.td_affine_clamp(g_.data_ptr(), n * c, 1, hh * ww, dtype_code(g_.dtype), mean_g.data_ptr(), std_g.data_ptr(),
                                      mean_x.data_ptr(), std_x.data_ptr(), lo.data_ptr(), hi.data_ptr(), current_stream_ptr(dev)))
        return g_

    # ------------------------------------------------------------------ kernel hijacks
    @torch.no_grad()
    @keep_signature
    def forward_one_step(self, x_in, sigma, **kwarg):
        """demofusion.py:185-214: skip-residual mix (c1), then the CFG forward with inner_model.forward patched."""
        p = self.p
        if self.is_kdiff:
            x_noisy = p.x + p.noise * sigma[0]
        else:
            a = p.sd_model.alphas_cumprod[self.timesteps[self.t_enc - p.current_step]]
            x_noisy = p.x * torch.sqrt(a) + p.noise * torch.sqrt(1 - a)
        self.cosine_factor = 0.5 * (1 + torch.cos(torch.pi * torch.tensor(((p.current_step + 1) / (self.t_enc + 1)))))
        c1 = self.cosine_factor ** p.cosine_scale_1
        x_in = x_in * (1 - c1) + x_noisy * c1
        jr = self.jitter_range if getattr(p, "random_jitter", False) and not self._wrap else 0   # a seamless canvas is not padded
        H, W = x_in.shape[2:]
        x_in_ = F.pad(x_in, (jr, jr, jr, jr), "constant", value=0) if jr else x_in      # demofusion.py:200-204
        cfg = self.sampler.model_wrap_cfg
        cfg.inner_model.forward = self.sample_one_step
        self.repeat_3 = False
        try:
            x_out = cfg.forward_ori(x_in_, sigma, **kwarg)
        finally:
            cfg.inner_model.forward = self.sampler_forward
        return x_out[:, :, jr:jr + H, jr:jr + W] if jr else x_out

    @torch.no_grad()
    @keep_signature
    def sample_one_step(self, x_in: Tensor, sigma: Tensor, cond):
        """demofusion.py:219-324.  With random jitter `x_in` is the latent zero-padded by jitter_range (the callers
        pad and crop: forward_one_step, get_noise), except on a seamless canvas (get_views' wrap_x / wrap_y)."""
        p = self.p
        sd_model = getattr(p, "sd_model", None) or self._sd_model()

        use_apply_model, self.repeat_3 = self.repeat_3, False   # demofusion.py:241-243

        def repeat_func(x_tile: Tensor, bboxes, mode=0) -> Tensor:
            n_rep = len(bboxes)
            if use_apply_model:
                return sd_model.apply_model(x_tile, sigma.repeat(n_rep), cond=self.repeat_cond_dict(cond, bboxes, mode))
            s_tile = self.repeat_tensor(sigma, n_rep)
            c_tile = self.repeat_cond_dict(cond, bboxes, mode) if isinstance(cond, dict) else self.repeat_tensor(cond, n_rep)
            return self.sampler_forward(x_tile, s_tile, cond=c_tile)

        x = self._check_input(x_in)
        N, C, H, W = x.shape
        jr = self.jitter_range if self._jitter and not self._wrap else 0     # the padding x_in carries
        if (H, W) != (self.h + 2 * jr, self.w + 2 * jr):
            raise ValueError(f"latent {(H, W)} does not match the views built for {(self.h, self.w)} (+ 2 x jitter {jr})")
        dt, dev = x.dtype, x.device
        s = int(p.current_scale_num)

        # ---- local windows: count-normalised blend (buffer in x.dtype / exact count, in fp32, rounded to x.dtype) ------
        if self._shard_on:
            x_local = self._local_pass_sharded(x, repeat_func)
            if x_local is None:
                return x_in
        elif self._jitter:
            x_local = self._local_pass_window_list(x_in, x, repeat_func)
            if x_local is None:
                return x_in
        else:
            if self._counts.device != dev:
                self._counts, self._rcp_counts = self._counts.to(dev), self._rcp_counts.to(dev)
            tiles = self._scatter_all(x)
            outs = []
            for batch_id, bboxes in enumerate(self.batched_bboxes):
                if host.interrupted():
                    return x_in
                outs.append(repeat_func(self._tile_batch(tiles, batch_id, N), bboxes))
            rcp = self._rcp_counts if dt in (torch.float16, torch.bfloat16) else None
            x_local = engine.blend_multidiffusion(self._grid, outs, N, C, self.tile_bs, self._counts, dt, flags=self._blend_flags,
                                                  rcp_weights=rcp).to(dt)

        # ---- blurred + renormalised latent for the global path ------------------------------------------------------
        c3 = 0.99 * self.cosine_factor ** p.cosine_scale_3 + 1e-2
        x_in_g = None
        if p.gaussian_filter:
            x_in_g = self._renormalise(self.gaussian_filter(x, kernel_size=2 * s - 1, sigma=self.sig * c3), x)
        elif not p.mixture:
            raise ValueError("DemoFusion without mixture needs gaussian_filter=True (the reference reads x_in_g unconditionally)")

        # ---- global dilated views ------------------------------------------------------------------------------------
        if self._wrap:     # views from 0 over the whole canvas
            end_y, end_x = H, W
        else:
            end = W - jr   # the reference's slice bound `end = shape[3] - jitter_range` is used on both axes
            end_y, end_x = min(H, end), end
        oh, ow = len(range(jr, end_y, s)), len(range(jr, end_x, s))
        if any(len(range(jr + b, end_y, s)) != oh for b in range(s)) or any(len(range(jr + b, end_x, s)) != ow for b in range(s)):
            raise ValueError("latent size must be a multiple of the scale (the reference's torch.cat needs equal views)")
        half = self.global_num_tiles // 2
        view_batches = self.local_global_batched_bboxes if self._shard_on else self.global_batched_bboxes
        g_outs, seen = [], (self._view_shard.begin if self._shard_on else 0)
        for bboxes in view_batches:
            n = len(bboxes)
            second = [1 if not (p.mixture and (seen + i) < half) else 0 for i in range(n)]
            seen += n
            view = engine.dilated_gather(x, x_in_g, [b[0] + jr for b in bboxes], [b[1] + jr for b in bboxes], second, s, oh, ow)
            g_outs.append(repeat_func(view, bboxes, mode=1).to(dt).contiguous())
        views_per_batch = self.global_tile_bs
        if self._shard_on:      # every rank needs every view's output: all-gather, one pointer-table entry per rank chunk
            g_outs = self._gather_chunks(g_outs, self._view_shard, N, (C, oh, ow), dt, dev)
            views_per_batch = self._view_shard.chunk

        # ---- add-back, /2, and the c2 mix: one launch ------------------------------------------------------------------
        c2 = float(self.cosine_factor ** p.cosine_scale_2)
        one_minus_c2 = float(1 - self.cosine_factor ** p.cosine_scale_2)
        out = engine.demofusion_combine(x_local, g_outs, views_per_batch, self.global_num_tiles, s, oh, ow, jr, end_y, end_x,
                                        bool(p.mixture), c2, one_minus_c2)
        self.x_buffer = out
        return out

    def _local_pass_sharded(self, x: Tensor, repeat_func):
        """Local windows with the tile shard: this rank scatters and denoises its chunk of the window list (grid or
        jittered), the outputs are all-gathered, every rank blends all windows.  None when interrupted."""
        N, C, H, W = x.shape
        dt, dev, ws, sh = x.dtype, x.device, self.window_size, self._shard
        outs = []
        if sh.num_local > 0:
            if self._jitter:
                if self._origins_dev.device != dev:
                    self._origins_dev = self._origins_dev.to(dev)
                host_part = (ctypes.c_int32 * (2 * sh.num_local))(*self._origins_host[2 * sh.begin:2 * sh.end])
                tiles = engine.scatter_bboxes(x, self._origins_dev[2 * sh.begin:2 * sh.end], host_part, sh.num_local, ws, ws,
                                              **self._list_wrap)
            else:
                tiles = engine.scatter_tiles(self._grid, x, tile_begin=sh.begin, tile_end=sh.end, flags=self._blend_flags)
            off = 0
            for bboxes in self.local_batched_bboxes:
                if host.interrupted():
                    return None
                outs.append(repeat_func(tiles[off * N:(off + len(bboxes)) * N], bboxes).to(dt).contiguous())
                off += len(bboxes)
        chunks = self._gather_chunks(outs, sh, N, (C, ws, ws), dt, dev)
        if self._jitter:
            return engine.blend_bboxes(chunks, sh.chunk, self._origins_dev, self._origins_host, self.num_tiles, N, C, H, W, ws, ws,
                                       **self._list_wrap).to(dt)
        if self._counts.device != dev:
            self._counts, self._rcp_counts = self._counts.to(dev), self._rcp_counts.to(dev)
        rcp = self._rcp_counts if dt in (torch.float16, torch.bfloat16) else None
        return engine.blend_multidiffusion(self._grid, chunks, N, C, sh.chunk, self._counts, dt, flags=self._blend_flags,
                                           rcp_weights=rcp).to(dt)

    def _local_pass_window_list(self, x_in: Tensor, x: Tensor, repeat_func):
        """Local windows in random-jitter mode (demofusion.py:254-264): one list-driven scatter, the UNet per batch, one
        list-driven count-normalised blend.  Returns x_local (x.dtype) or None when interrupted."""
        N, C, H, W = x.shape
        dt, dev, ws, T = x.dtype, x.device, self.window_size, self.num_tiles
        if self._origins_dev.device != dev:
            self._origins_dev = self._origins_dev.to(dev)
        self._tiles = engine.scatter_bboxes(x, self._origins_dev, self._origins_host, T, ws, ws, out=self._tiles, **self._list_wrap)
        outs = []
        for batch_id, bboxes in enumerate(self.batched_bboxes):
            if host.interrupted():
                return None
            outs.append(repeat_func(self._tile_batch(self._tiles, batch_id, N), bboxes).to(dt).contiguous())
        return engine.blend_bboxes(outs, self.tile_bs, self._origins_dev, self._origins_host, T, N, C, H, W, ws, ws,
                                   **self._list_wrap).to(dt)

    def get_noise(self, x_in: Tensor, sigma_in: Tensor, cond_in: Dict[str, Tensor], step: int) -> Tensor:
        """demofusion.py:345-353: the tiled eps on the latent padded by jitter_range, cropped back (never padded on a
        seamless canvas)."""
        self.repeat_3 = True
        self.cosine_factor = 0.5 * (1 + torch.cos(torch.pi * torch.tensor(((self.p.current_step + 1) / (self.t_enc + 1)))))
        jr = 0 if self._wrap else self.jitter_range
        if not jr:
            return self.sample_one_step(x_in, sigma_in, cond_in.copy())
        H, W = x_in.shape[2:]
        x_in_ = F.pad(x_in, (jr, jr, jr, jr), "constant", value=0)
        return self.sample_one_step(x_in_, sigma_in, cond_in.copy())[:, :, jr:jr + H, jr:jr + W]
