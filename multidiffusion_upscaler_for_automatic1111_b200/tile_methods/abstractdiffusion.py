"""Base tile-method delegate with the reference's surface
(tile_methods/abstractdiffusion.py), H100-native underneath.

What differs from the reference by design:
  * `init_grid_bbox` also builds a `td_grid` plan (C-ABI) and a persistent
    tile-batch buffer: the whole step's scatter is ONE kernel launch and the
    UNet receives views of that buffer (the tile batch is small next to 80 GB of HBM: no need to re-cat).
  * `reset_buffer` only (re)allocates: the fused gather-form blend writes every
    canvas pixel, so the per-step `zero_()` pass of the reference is not needed.
  * Region prompt control (SURVEY.md section 8(f)-1) is built on the same kernels: the grid tiles go through the
    fused blend (which then also returns the un-normalised `x_buffer`), the handful of custom regions are cropped,
    added and feather-composited with the reference's own tensor expressions.
  * ControlNet / StableSR tile caches (section 8(f)-2) are the scatter kernel applied to the side inputs: one launch
    per hint on the tile plan scaled to pixel space, the per-batch caches are views of that one tensor.
  * Tiled noise inversion (section 8(f)-3) is the Euler inversion loop of the reference around our tiled `get_noise`.
"""
from __future__ import annotations

import ctypes
import math
from types import MethodType
from typing import Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from .. import engine, host
from ..host import opt_f
from ..tile_utils.utils import (BBox, BlendMode, Condition, CustomBBox, Prompt, custom_bbox, custom_bbox_rect, get_retouch_mask,
                                grid_bbox, keep_signature, noise_inverse, controlnet, stablesr)

CondDict = Dict[str, Union[Tensor, List[Tensor]]]

_MASK_DTYPES = (torch.float16, torch.bfloat16, torch.float32)


class InpaintPlan:
    """What `init_inpaint_mask` leaves on a delegate: the grid tiles and custom regions the inpaint mask reaches and the compact
    tile batches of the sampler loop (active tiles in tile order, `tile_bs` per batch)."""

    def __init__(self, g, active: np.ndarray, regions: List[bool], tile_bs: int, device):
        self.active = active                                   # bool [T]
        self.tiles = [int(t) for t in np.flatnonzero(active)]  # active tile indices, ascending
        self.slot_host = engine.slot_table(active)             # int32 [T]: compact position or -1
        self.slot_dev = torch.from_numpy(self.slot_host).to(device)
        xywh = engine.grid_bboxes_xywh(g) if g is not None else np.zeros((0, 4), dtype=np.int32)
        bboxes = [BBox(*(int(v) for v in xywh[t])) for t in self.tiles]
        self.batched_bboxes = [bboxes[i:i + tile_bs] for i in range(0, len(bboxes), tile_bs)]
        flat = [int(v) for t in self.tiles for v in xywh[t, :2]]          # (x, y) per active tile
        self.origins_host = (ctypes.c_int32 * max(1, len(flat)))(*flat)
        self.origins_dev = torch.tensor(flat, dtype=torch.int32, device=device)
        self.regions = regions                                 # per custom region: denoised (True) or skipped

    @property
    def num_tiles(self) -> int:
        return len(self.tiles)


class AbstractDiffusion:

    def __init__(self, p, sampler):
        self.method = self.__class__.__name__
        self.p = p
        self.pbar = None

        # sampler (abstractdiffusion.py:11-14)
        self.sampler_name = p.sampler_name
        self.sampler_raw = sampler
        self.sampler = sampler

        # image-editing (ip2p) models add one more cond slot (abstractdiffusion.py:16-20)
        if self.is_kdiff and not hasattr(self, "is_edit_model"):
            sd_model = self._sd_model()
            cfg = getattr(self.sampler, "model_wrap_cfg", None)
            scale = getattr(cfg, "image_cfg_scale", None)
            self.is_edit_model = (getattr(sd_model, "cond_stage_key", None) == "edit"
                                  and scale is not None and scale != 1.0)

        # latent canvas + persistent state (abstractdiffusion.py:22-28)
        self.x_buffer: Optional[Tensor] = None
        self.w: int = int(self.p.width // opt_f)
        self.h: int = int(self.p.height // opt_f)
        self.weights: Tensor = torch.zeros((1, 1, self.h, self.w), device=host.device(), dtype=torch.float32)

        self.step_count = 0
        self.inner_loop_count = 0
        self.kdiff_step = -1

        # grid tiling (abstractdiffusion.py:35-42)
        self.enable_grid_bbox: bool = False
        self.tile_w: Optional[int] = None
        self.tile_h: Optional[int] = None
        self.tile_bs: Optional[int] = None
        self.num_tiles: Optional[int] = None
        self.num_batches: Optional[int] = None
        self.batched_bboxes: List[List[BBox]] = []

        # region prompt control (abstractdiffusion.py:44-49)
        self.enable_custom_bbox: bool = False
        self.custom_bboxes: List[CustomBBox] = []
        self.cond_basis = None
        self.uncond_basis = None
        self.draw_background: bool = True
        self.causal_layers: Optional[bool] = None

        # tiled noise inversion (abstractdiffusion.py:52-60)
        self.noise_inverse_enabled: bool = False
        self.noise_inverse_steps: Optional[int] = None
        self.noise_inverse_retouch: Optional[float] = None
        self.noise_inverse_renoise_strength: Optional[float] = None
        self.noise_inverse_renoise_kernel: Optional[int] = None
        self.noise_inverse_get_cache = None
        self.noise_inverse_set_cache = None
        self.sample_img2img_original = None

        # ext. ControlNet / StableSR side inputs (abstractdiffusion.py:62-75)
        self.enable_controlnet: bool = False
        self.controlnet_script = None
        self.control_tensor_batch = None
        self.control_params = None
        self.control_tensor_cpu: bool = False
        self.control_tensor_custom: list = []
        self.enable_stablesr: bool = False
        self.stablesr_script = None
        self.stablesr_tensor: Optional[Tensor] = None
        self.stablesr_tensor_batch = None
        self.stablesr_tensor_custom: list = []

        # device engine state
        self._grid = None                     # td_grid plan
        self._tiles: Optional[Tensor] = None  # persistent [T*N, C, th, tw] scatter target
        self._icond_tiles: Optional[Tensor] = None
        self._blend_flags = 0                 # tests flip TD_FLAG_FORCE_GENERIC here
        self._rcp_weights: Optional[Tensor] = None   # RN(1/weights) when all weights are small integers
        self._shard = None                    # parallel.TileShard when tiles are sharded over ranks
        self._shard_group = None
        self._shard_fused = False
        self._exchange = None                 # parallel.PeerExchange (fused path)
        self._shard_step = 0
        self._shard_mode = "replicate"
        self._strip = None
        self._strip_exchange = None
        self._region_shard = None             # parallel.RegionShard: custom regions under the tile shard
        self._inpaint: Optional[InpaintPlan] = None   # init_inpaint_mask: the tiles and regions the sampler loop denoises
        self._full_plan_pass = False          # tiled noise inversion: every tile and region, whatever the inpaint mask

    # ----------------------------------------------------------------- helpers
    def _sd_model(self):
        m = getattr(host.get_shared(), "sd_model", None)
        return m if m is not None else getattr(self.p, "sd_model", None)

    @property
    def is_kdiff(self) -> bool:
        return host.is_kdiff_sampler(self.sampler_raw)

    @property
    def is_ddim(self) -> bool:
        return host.is_ddim_sampler(self.sampler_raw)

    def update_pbar(self):
        if self.pbar is None:
            return
        if self.pbar.n >= self.pbar.total:
            self.pbar.close()
            return
        st = host.get_shared().state
        if self.step_count == st.sampling_step:
            self.inner_loop_count += 1
            if self.inner_loop_count < self.total_bboxes:
                self.pbar.update()
        else:
            self.step_count = st.sampling_step
            self.inner_loop_count = 0

    def reset_buffer(self, x_in: Tensor):
        """abstractdiffusion.py:97-102.  Allocation only -- the blend kernel overwrites every pixel."""
        if self.x_buffer is None or self.x_buffer.shape != x_in.shape or self.x_buffer.dtype != x_in.dtype \
                or self.x_buffer.device != x_in.device:
            self.x_buffer = torch.zeros_like(x_in)

    def init_done(self):
        """abstractdiffusion.py:104-117: sanity check + progress accounting."""
        self._init_rcp_weights()
        self.total_bboxes = 0
        if self.enable_grid_bbox:
            self.total_bboxes += self.num_batches
        if self.enable_custom_bbox:
            self.total_bboxes += len(self.custom_bboxes)
        assert self.total_bboxes > 0, "Nothing to paint! No background to draw and no custom bboxes were provided."
        if self._inpaint is not None:       # progress counts the denoiser calls the sampler loop makes
            self.total_bboxes = (len(self._inpaint.batched_bboxes) if self.enable_grid_bbox else 0) + \
                (sum(self._inpaint.regions) if self.enable_custom_bbox else 0)
        self.pbar = None
        if getattr(self.p, "show_tile_progress", False):
            from tqdm import tqdm
            steps = getattr(host.get_shared().state, "sampling_steps", 1)
            self.pbar = tqdm(total=self.total_bboxes * steps, desc=f"{self.method} Sampling: ")

    def _init_rcp_weights(self):
        """RN(1/weights) of the job's weight canvas for the blend's exact fast divide, or None when the canvas does not qualify."""
        rcp = engine.exact_reciprocals(self.weights.detach().to("cpu", torch.float32).numpy().reshape(self.h, self.w))
        self._rcp_weights = None if rcp is None else torch.from_numpy(rcp).to(self.weights.device)

    # ------------------------------------------------------- cond-dict access
    def _tcond_key(self, cond_dict: CondDict) -> str:
        return "crossattn" if "crossattn" in cond_dict else "c_crossattn"

    def get_tcond(self, cond_dict: CondDict) -> Tensor:
        tcond = cond_dict[self._tcond_key(cond_dict)]
        return tcond[0] if isinstance(tcond, list) else tcond

    def set_tcond(self, cond_dict: CondDict, tcond: Tensor):
        key = self._tcond_key(cond_dict)
        cond_dict[key] = [tcond] if isinstance(cond_dict[key], list) else tcond

    def _icond_key(self, cond_dict: CondDict) -> str:
        # the model's conditioning key cannot change during a job: resolved once per model object (this sits on the
        # per-tile-batch path, 25 batches x 3 lookups per sampler step at the UI default)
        sd_model = self._sd_model()
        cached = self.__dict__.get("_icond_key_cache")
        if cached is not None and cached[0] is sd_model:
            return cached[1]
        ck = getattr(getattr(sd_model, "model", None), "conditioning_key", None)
        key = "c_adm" if ck in ("crossattn-adm", "adm") else "c_concat"
        self._icond_key_cache = (sd_model, key)
        return key

    def get_icond(self, cond_dict: CondDict) -> Tensor:
        icond = cond_dict[self._icond_key(cond_dict)]
        return icond[0] if isinstance(icond, list) else icond

    def set_icond(self, cond_dict: CondDict, icond: Tensor):
        key = self._icond_key(cond_dict)
        cond_dict[key] = [icond] if isinstance(cond_dict[key], list) else icond

    def _vcond_key(self, cond_dict: CondDict) -> Optional[str]:
        return "vector" if "vector" in cond_dict else None

    def get_vcond(self, cond_dict: CondDict) -> Optional[Tensor]:
        return cond_dict.get(self._vcond_key(cond_dict))

    def set_vcond(self, cond_dict: CondDict, vcond: Optional[Tensor]):
        key = self._vcond_key(cond_dict)
        if key is not None:
            cond_dict[key] = vcond

    def make_cond_dict(self, cond_in: CondDict, tcond: Tensor, icond: Tensor, vcond: Tensor = None) -> CondDict:
        cond_out = cond_in.copy()
        self.set_tcond(cond_out, tcond)
        self.set_icond(cond_out, icond)
        self.set_vcond(cond_out, vcond)
        return cond_out

    # ------------------------------------------------------------ grid tiling
    @grid_bbox
    def init_grid_bbox(self, tile_w: int, tile_h: int, overlap: int, tile_bs: int, wrap_x: bool = False, wrap_y: bool = False):
        """abstractdiffusion.py:172-186, bookkeeping done by td_grid_init (C++, bit-exact).

        wrap_x / wrap_y make the canvas periodic on that axis (seamless output: panoramas that close on themselves,
        repeating textures).  The tiles are then spaced evenly around the circle and the last ones run past the edge
        and continue at 0, so the blend mixes both sides of the seam.  On a wrapped axis a grid
        BBox may therefore end past the canvas (x + w > W): its `slicer` is not a crop of the latent, every grid-tile
        crop goes through the engine, which reads the plan's wrap bits."""
        wrap = (engine.WRAP_X if wrap_x else 0) | (engine.WRAP_Y if wrap_y else 0)
        if wrap and self.method == "DemoFusion":
            raise NotImplementedError("DemoFusion builds its own window lists: pass wrap_x / wrap_y to DemoFusion.get_views(...)")
        self.enable_grid_bbox = True
        g = engine.make_grid(self.w, self.h, tile_w, tile_h, overlap, tile_bs, wrap=wrap)
        self._grid = g
        self.tile_w, self.tile_h = int(g.tile_w), int(g.tile_h)
        tile_weights = self.get_tile_weights()
        tw_np = None
        if isinstance(tile_weights, Tensor):
            tw_np = tile_weights.detach().to("cpu", torch.float32).numpy()
        elif float(tile_weights) != 1.0:
            raise ValueError("scalar tile weights other than 1.0 are not part of the reference")
        weights = engine.grid_weights(g, tw_np)
        self.weights += torch.from_numpy(weights).view(1, 1, self.h, self.w).to(self.weights.device)
        self._set_grid_bboxes(g)

    def _set_grid_bboxes(self, g):
        """num_tiles, num_batches, tile_bs and batched_bboxes of the tile plan g."""
        bboxes = [BBox(int(x), int(y), int(w), int(h)) for x, y, w, h in engine.grid_bboxes_xywh(g)]
        self.num_tiles = len(bboxes)
        self.num_batches = int(g.num_batches)
        self.tile_bs = int(g.tile_bs)
        self.batched_bboxes = [bboxes[i * self.tile_bs:(i + 1) * self.tile_bs] for i in range(self.num_batches)]

    @grid_bbox
    def get_tile_weights(self) -> Union[Tensor, float]:
        return 1.0

    # ------------------------------------------------------------- inpainting
    def init_inpaint_mask(self, mask: Tensor):
        """Denoise only the grid tiles and custom regions the inpaint mask reaches.  Call after init_grid_bbox / init_custom_bbox
        and before init_done.

        `mask` is the WebUI's latent mask `p.mask` (1 = keep the original): [h, w], [C, h, w] or [N, C, h, w], fp16 / bf16 /
        fp32, on the device.  A tile (region) is active when at least one mask element in its window (rectangle), over all
        leading planes, is not exactly 1.0 -- NaN included.  The other tiles cannot change a pixel the host keeps: their windows
        lie in the kept area, which the host overwrites with the original after every denoiser call.  The weight canvas and the
        Mixture of Diffusers rescale factor stay those of the full plan, so on every pixel with mask < 1 the step computes what
        the full plan computes, visiting the same tiles in the same order.  A mask that keeps everything leaves nothing to
        denoise: the step then returns the blend of nothing (zeros).  Tiled noise inversion (`get_noise`) still runs every tile.

        With a UNet whose output for one sample depends on the batch it runs in, results differ in the last bits, as they do
        for another tile_bs: the active tiles are batched differently."""
        self._refuse_inpaint()
        if not isinstance(mask, Tensor) or mask.dim() not in (2, 3, 4) or tuple(mask.shape[-2:]) != (self.h, self.w):
            raise ValueError(f"{self.method}: the inpaint mask must be [h, w], [C, h, w] or [N, C, h, w] with (h, w) = {(self.h, self.w)}, "
                             f"got {tuple(mask.shape) if isinstance(mask, Tensor) else type(mask).__name__}")
        if mask.dtype not in _MASK_DTYPES:
            raise ValueError(f"{self.method}: the inpaint mask must be fp16, bf16 or fp32, got {mask.dtype}")
        grid = self._grid if self.enable_grid_bbox else None
        active = engine.active_tiles(grid, mask) if grid is not None else np.zeros(0, dtype=bool)
        regions = [bool(engine.active_tiles(engine.rect_grid(self.w, self.h, b.x, b.y, b.w, b.h), mask)[0]) for b in self.custom_bboxes]
        self._inpaint = InpaintPlan(grid, active, regions, self.tile_bs or 1, mask.device)
        # side-input caches built before this call hold the full plan's tiles
        if self.control_tensor_batch is not None:
            self.prepare_controlnet_tensors(refresh=True)
        if self.stablesr_tensor is not None:
            self.stablesr_tensor_batch, _ = self._side_input_tiles(self.stablesr_tensor, 1, False)

    def _refuse_inpaint(self):
        """NotImplementedError for a plan init_inpaint_mask has no form for (raised before any state changes)."""
        if self._grid is not None and self._grid.wrap:
            raise NotImplementedError(f"{self.method}: init_inpaint_mask() does not take a wrapped plan (wrap_x / wrap_y)")
        if self._shard is not None:
            raise NotImplementedError(f"{self.method}: init_inpaint_mask() does not run under the multi-GPU tile shard")

    def _active_plan(self) -> Optional[InpaintPlan]:
        """The inpaint plan the sampler loop runs, or None for the full plan."""
        return None if self._full_plan_pass else self._inpaint

    def _region_skipped(self, bbox_id: int) -> bool:
        ip = self._active_plan()
        return ip is not None and not ip.regions[bbox_id]

    def _scatter_active(self, x: Tensor, ip: InpaintPlan) -> Tensor:
        """The active tiles of x, compact and in tile order (td_scatter_bboxes: the same copy as td_scatter_tiles)."""
        self._tiles = engine.scatter_bboxes(x, ip.origins_dev, ip.origins_host, ip.num_tiles, self.tile_h, self.tile_w, out=self._tiles)
        return self._tiles

    # ------------------------------------------------------------- multi-GPU
    def init_tile_shard(self, group=None, fused: bool = True, mode: Optional[str] = None):
        """Shard the tiles over the ranks of `group` (one process per GPU).  Call after init_grid_bbox.

        mode "strip" (default with fused=True for MultiDiffusion): rank r denoises a contiguous run of tile ROWS and
        blends only the canvas rows it owns; per step only the overlapping tile rows go to the next rank(s) and the
        rows of the blended latent the previous rank(s) scatter from come back (parallel.StripShard / StripExchange:
        pushed over NVLink into CUDA-IPC-mapped buffers, flag-synchronised, no NCCL on the data path).  The tensor
        `sample_one_step` returns is valid on the rank's own rows plus that halo; `gather_latent` assembles the full
        latent (after the last step).  Bit-identical to a single-GPU run.
        mode "replicate": each rank denoises `tiles[begin:end)`, ALL tile outputs are exchanged (fused: peer reads over
        NVLink inside the blend kernel; else NCCL all-gather) and every rank blends the full latent.

        Custom regions (init_custom_bbox) are shared out as well: region j is denoised by rank j % world and its output
        all-gathered (parallel.RegionShard); in strip mode its input rows are gathered from the strips' owners first.  Every
        rank composites the regions over the rows it returns.  Without a background layer (draw_background=False, no
        init_grid_bbox) only the regions are sharded, in replicate mode.

        A wrapped grid (init_grid_bbox(..., wrap_x / wrap_y), seamless tiling) needs an explicit mode: under "strip" with
        wrap_y the strips close into a ring (StripShard(wrap_y=True)); both modes stay bit-identical to one GPU."""
        import torch.distributed as dist
        from .. import parallel
        if self._inpaint is not None:
            raise NotImplementedError(f"{self.method}: init_tile_shard() does not run with an inpaint mask (init_inpaint_mask)")
        if self._grid is None and not self.enable_custom_bbox:
            raise RuntimeError("init_tile_shard() must follow init_grid_bbox() or init_custom_bbox()")
        if self._grid is not None and self._grid.wrap and mode is None:
            raise NotImplementedError("init_tile_shard() on a wrapped grid (wrap_x / wrap_y, a periodic canvas) needs an explicit "
                                      "mode='strip' or mode='replicate'")
        if mode is None:
            mode = "strip" if (fused and self.method == "MultiDiffusion" and self._grid is not None) else "replicate"
        if mode not in ("strip", "replicate"):
            raise ValueError(f"unknown shard mode {mode!r}")
        if mode == "strip" and self._grid is None:
            raise ValueError("the strip shard partitions the grid tiles: it needs init_grid_bbox()")
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        self._shard_group, self._shard_fused, self._shard_mode = group, fused, mode
        self._region_shard = None
        bboxes = [b for batch in self.batched_bboxes for b in batch]
        g = self._grid
        if g is None:
            self._strip = None
            self._shard = parallel.TileShard(0, rank, world)
        elif mode == "strip":
            self._strip = parallel.StripShard(list(g.ys[:g.rows]), g.cols, g.tile_h, g.H, rank, world,
                                              wrap_y=bool(g.wrap & engine.WRAP_Y))
            t0, t1 = self._strip.tile_range()
            self._shard = parallel.TileShard(self.num_tiles, rank, world)     # kept for callers that read .begin / .end
            self._shard.begin, self._shard.end = t0, t1
        else:
            self._strip = None
            self._shard = parallel.TileShard(self.num_tiles, rank, world)
        local = bboxes[self._shard.begin:self._shard.end]
        self.local_batched_bboxes = [local[i:i + self.tile_bs] for i in range(0, len(local), self.tile_bs)] if local else []
        return self._shard

    def gather_latent(self, x: Tensor) -> Tensor:
        """Strip shard: the full latent from every rank's rows of `x` (call once, after the last sampler step).
        Other modes keep the latent replicated: returns x."""
        if getattr(self, "_strip", None) is None or self._strip_exchange is None:
            return x
        return self._strip_exchange.gather_latent(x)

    def _strip_step(self, outs, x: Tensor, N: int, C: int, regions_done=None) -> Tensor:
        """Strip-shard tail of a sharded step (MultiDiffusion and Mixture of Diffusers): own tile outputs -> halo push -> strip
        blend (`_strip_blend`; with regions into the accumulator x_buffer) -> region composite of the own rows -> latent halo.
        Returns the exchange's latent buffer, valid on the strip and its latent halo."""
        from .. import parallel
        g = self._grid
        if self._strip_exchange is None:
            self._strip_exchange = parallel.StripExchange(self._strip, N, C, g.tile_w, g.W, x.dtype, x.device, self._shard_group,
                                                          latent_dtype=self._strip_latent_dtype(x.dtype))
        ex = self._strip_exchange
        if ex.N != N or ex.dtype != x.dtype:
            raise ValueError(f"row-strip shard: the exchange was built for N={ex.N}, {ex.dtype}; this step has N={N}, {x.dtype}")
        lo, hi = self._strip.strip()
        x_out = ex.x_out
        if self.enable_grid_bbox:
            own = ex.own_tiles()
            off = 0
            for o in outs:
                own[off:off + o.shape[0]].copy_(o)
                off += o.shape[0]
            ex.push_tile_halos()
            self._strip_blend(ex, x, self.x_buffer if regions_done is not None else None)
        else:
            # draw_background=False: no grid pass, the regions paint over zeros (the tile halos are not exchanged at all)
            self.x_buffer[:, :, lo:hi].zero_()
        if regions_done is not None:
            weights, background_aux = self._region_composite_terms()
            if x_out.dtype == torch.float32:
                self._composite_regions(self.x_buffer, weights, regions_done, background_aux, rows=(lo, hi), out=x_out)
            else:        # the composite writes fp32; BACKGROUND-only results are values of the latent dtype (lossless copy)
                if getattr(self, "_strip_composite_f32", None) is None or self._strip_composite_f32.shape != x_out.shape:
                    self._strip_composite_f32 = torch.empty(x_out.shape, dtype=torch.float32, device=x_out.device)
                f32 = self._composite_regions(self.x_buffer, weights, regions_done, background_aux, rows=(lo, hi),
                                              out=self._strip_composite_f32)
                x_out[:, :, lo:hi].copy_(f32[:, :, lo:hi])
        ex.push_x_halos_and_wait()
        return x_out

    def _strip_latent_dtype(self, x_dtype: torch.dtype) -> torch.dtype:
        """Dtype of the latent a strip step returns (and of the exchange's latent buffer)."""
        raise NotImplementedError(f"{self.method} has no row-strip shard")

    def _strip_blend(self, ex, x: Tensor, x_buffer: Optional[Tensor]):
        """Blend this rank's strip (the exchange's latent buffer; with `x_buffer` also / instead the accumulator there)."""
        raise NotImplementedError(f"{self.method} has no row-strip shard")

    def _region_composite_terms(self):
        """(weights, background_aux) of `_composite_regions` for this method."""
        raise NotImplementedError(f"{self.method} has no region composite")

    def _region_pass_sharded(self, x: Tensor, custom_func: Callable, poll_interrupt: bool, interrupted: bool):
        """`_custom_region_pass` under the tile shard: this rank denoises its regions (parallel.RegionShard: region j on rank
        j % world), whose inputs come from the local latent (replicate mode) or from the strips' owners (strip mode, one
        all-gather), and one all-gather of the outputs gives every rank every region output.  An interrupted rank still
        takes part in both exchanges with placeholder outputs (its inputs) so that the collectives stay in lock-step.

        Returns ([(bbox_id, bbox, x_tile_out)] in list order, interrupted)."""
        from .. import parallel
        if self._region_shard is None:
            self._region_shard = parallel.RegionShard([(b.x, b.y, b.w, b.h) for b in self.custom_bboxes], self._shard.rank,
                                                      self._shard.world)
        rs = self._region_shard
        if self._strip is not None:
            inputs = parallel.gather_region_inputs(rs, x, self._strip.B, self._shard_group)
        else:
            inputs = {j: x[self.custom_bboxes[j].slicer] for j in rs.mine()}
        use_networks = not getattr(self.p, "disable_extra_networks", False)
        outs = []
        for j in rs.mine():
            bbox = self.custom_bboxes[j]
            if interrupted or (poll_interrupt and host.interrupted()):
                interrupted = True
                outs.append(inputs[j])          # placeholder with the right shape: the exchange must still happen
                continue
            if use_networks:
                host.extra_networks_activate(self.p, bbox.extra_network_data)
            outs.append(custom_func(inputs[j], j, bbox))
            if use_networks:
                host.extra_networks_deactivate(self.p, bbox.extra_network_data)
            self.update_pbar()
        all_outs = parallel.exchange_region_outputs(rs, outs, x, self._shard_group)
        return [(j, b, all_outs[j]) for j, b in enumerate(self.custom_bboxes)], interrupted

    def _exchange_and_blend_md(self, outs, x: Tensor, N: int, C: int, x_buffer: Optional[Tensor] = None) -> Tensor:
        """Tile-shard tail of MultiDiffusion.sample_one_step (`x_buffer`: also store the un-normalised accumulator there)."""
        from .. import parallel
        sh, g = self._shard, self._grid
        plane = N * C * g.tile_h * g.tile_w
        dt = outs[0].dtype if outs else x.dtype
        self._shard_step += 1
        if self._shard_fused:
            if self._exchange is None:
                self._exchange = parallel.PeerExchange(sh.chunk * plane * x.element_size(), x.device, self._shard_group)
            parity = self._shard_step & 1
            if outs:
                buf = self._exchange.local_buffer(parity, dt)[:sh.num_local * plane].view(sh.num_local * N, C, g.tile_h, g.tile_w)
                torch.cat([o.to(dt) for o in outs], dim=0, out=buf)
            self._exchange.signal()
            return parallel.blend_multidiffusion_peer(g, self._exchange, parity, sh, N, C, self.weights, dt, x_buffer=x_buffer)
        local = torch.zeros((sh.chunk * N, C, g.tile_h, g.tile_w), dtype=dt, device=x.device)
        if outs:
            torch.cat(outs, dim=0, out=local[:sh.num_local * N])
        gathered = parallel.gather_tile_outputs(local, self._shard_group)
        chunks = []
        for b in range(sh.num_chunks):
            nt = min(sh.chunk, sh.num_tiles - b * sh.chunk)
            chunks.append(gathered[b * sh.chunk * N: (b * sh.chunk + nt) * N])
        return engine.blend_multidiffusion(g, chunks, N, C, sh.chunk, self.weights, x.dtype, x_buffer=x_buffer, flags=self._blend_flags,
                                           rcp_weights=self._rcp_weights)

    # ------------------------------------------------- region prompt control
    @custom_bbox
    def init_custom_bbox(self, bbox_settings: Dict[int, tuple], draw_background: bool, causal_layers: bool):
        """abstractdiffusion.py:193-229: region rectangles in latent units (td_custom_bbox_rect, bit-exact with the
        reference's float64 arithmetic) and their prompt conditionings (host application's prompt parser)."""
        self.enable_custom_bbox = True
        self.causal_layers = causal_layers
        self.draw_background = draw_background
        if not draw_background:
            self.enable_grid_bbox = False
            self.weights.zero_()

        self.custom_bboxes = []
        for setting in bbox_settings.values():
            e, x, y, w, h, prompt, neg_prompt, blend_mode, feather_ratio, seed = setting
            if not e:
                continue
            rect = custom_bbox_rect(x, y, w, h, self.w, self.h)
            if rect is None:
                continue
            self.custom_bboxes.append(CustomBBox(*rect, prompt, neg_prompt, blend_mode, feather_ratio, seed))

        if len(self.custom_bboxes) == 0:
            self.enable_custom_bbox = False
            return

        if host.a1111_module("prompt_parser") is None:
            # no text encoder outside the WebUI: the caller's `custom_func` owns the conditioning
            return
        p = self.p
        prompts = p.all_prompts[:p.batch_size]
        neg_prompts = p.all_negative_prompts[:p.batch_size]
        for bbox in self.custom_bboxes:
            bbox.cond, bbox.extra_network_data = Condition.get_custom_cond(prompts, bbox.prompt, p.steps, p.styles)
            bbox.uncond = Condition.get_uncond(Prompt.append_prompt(neg_prompts, bbox.neg_prompt), p.steps, p.styles)
        self.cond_basis = Condition.get_cond(prompts, p.steps)
        self.uncond_basis = Condition.get_uncond(neg_prompts, p.steps)

    @custom_bbox
    def reconstruct_custom_cond(self, org_cond: CondDict, custom_cond, custom_uncond, bbox: CustomBBox):
        """abstractdiffusion.py:231-243: the region's text cond / uncond at the sampler's current step, and the
        image cond cropped to the region when it is spatial (img2img)."""
        image_conditioning = None
        if isinstance(org_cond, dict):
            icond = self.get_icond(org_cond)
            if tuple(icond.shape[2:]) == (self.h, self.w):
                icond = icond[bbox.slicer]
            image_conditioning = icond
        step = self.sampler.model_wrap_cfg.step
        return Condition.reconstruct_cond(custom_cond, step), Condition.reconstruct_uncond(custom_uncond, step), image_conditioning

    def _forward_region(self, bbox_id: int, forward_func: Callable, x: Tensor, sigma: Tensor, original_cond: CondDict,
                        tcond: Tensor, icond) -> Tensor:
        self.set_custom_controlnet_tensors(bbox_id, x.shape[0])
        self.set_custom_stablesr_tensors(bbox_id)
        return forward_func(x, sigma, cond=self.make_cond_dict(original_cond, tcond, icond))

    def _forward_region_split(self, bbox_id: int, forward_func: Callable, x_tile: Tensor, sigma_in: Tensor, original_cond: CondDict,
                              first: Tensor, second: Tensor, icond_first, icond_second, pad_with_second: bool = False) -> Tensor:
        """Two UNet calls when the cond and uncond token counts differ (they cannot share a batch):
        rows [0, n1) with `first`, the next n2 rows with `second` (abstractdiffusion.py:288-311, :376-395)."""
        x_out = torch.zeros_like(x_tile)
        n1, n2 = first.shape[0], second.shape[0]
        out1 = self._forward_region(bbox_id, forward_func, x_tile[:n1], sigma_in[:n1], original_cond, first, icond_first)
        hi = n1 + n2 if pad_with_second else x_tile.shape[0]
        out2 = self._forward_region(bbox_id, forward_func, x_tile[n1:hi], sigma_in[n1:hi], original_cond, second, icond_second)
        x_out[:n1] = out1
        x_out[n1:hi] = out2
        if pad_with_second and self.is_edit_model:
            x_out[hi:] = out2
        return x_out

    @custom_bbox
    def kdiff_custom_forward(self, x_tile: Tensor, sigma_in: Tensor, original_cond: CondDict, bbox_id: int, bbox: CustomBBox,
                             forward_func: Callable) -> Tensor:
        """Denoise one custom region the way the k-diffusion CFG wrapper batches the whole image
        (abstractdiffusion.py:245-427).  The wrapper feeds [cond rows, uncond rows(, uncond rows for edit models)]
        either in one batch or -- low-VRAM mode, or prompts of different token length -- in slices; the region's
        own cond / uncond have to be fed in the same row layout."""
        step = self.sampler.model_wrap_cfg.step
        if self.kdiff_step != step:                       # a new sampler step: forget per-step state
            self.kdiff_step = step
            self.kdiff_step_bbox = [-1] * len(self.custom_bboxes)
            self.tensor, self.uncond, self.image_cond_in = {}, {}, {}
            # the global prompts tell how the wrapper batches this step
            self.real_tensor = Condition.reconstruct_cond(self.cond_basis, step)
            self.real_uncond = Condition.reconstruct_uncond(self.uncond_basis, step)
            self.a = [0] * len(self.custom_bboxes)        # rows of the virtual batch already served, per region
        same_len_global = self.real_tensor.shape[1] == self.real_uncond.shape[1]

        if self.kdiff_step_bbox[bbox_id] != step:         # first call for this region in this step
            self.kdiff_step_bbox[bbox_id] = step
            tensor, uncond, icond = self.reconstruct_custom_cond(original_cond, bbox.cond, bbox.uncond, bbox)
            if same_len_global and host.batch_cond_uncond():
                # x_tile holds the complete virtual batch
                if tensor.shape[1] == uncond.shape[1]:
                    parts = [tensor, uncond, uncond] if self.is_edit_model else [tensor, uncond]
                    return self._forward_region(bbox_id, forward_func, x_tile, sigma_in, original_cond, torch.cat(parts), icond)
                n1, n2 = tensor.shape[0], uncond.shape[0]
                return self._forward_region_split(bbox_id, forward_func, x_tile, sigma_in, original_cond, tensor, uncond,
                                                  icond[:n1], icond[n1:n1 + n2], pad_with_second=True)
            # x_tile is a slice of the virtual batch: keep the region's tensors for the following calls
            self.tensor[bbox_id], self.uncond[bbox_id], self.image_cond_in[bbox_id] = tensor, uncond, icond

        tensor, uncond, icond = self.tensor[bbox_id], self.uncond[bbox_id], self.image_cond_in[bbox_id]
        a = self.a[bbox_id]
        b = a + x_tile.shape[0]
        self.a[bbox_id] = b
        T, U = tensor.shape[0], uncond.shape[0]

        if same_len_global:
            # rows [a, b) of the virtual batch [tensor | uncond (| uncond)]
            segments = [(tensor, 0)] + [(uncond, T + k * U) for k in range(2 if self.is_edit_model else 1)]
            cond_rows, uncond_rows = [], []
            for seg, lo in segments:
                s, e = max(a, lo) - lo, min(b, lo + seg.shape[0]) - lo
                if e > s:
                    (cond_rows if seg is tensor else uncond_rows).append(seg[s:e])
            if not cond_rows:                              # the slice lies entirely in the uncond rows
                return self._forward_region(bbox_id, forward_func, x_tile, sigma_in, original_cond,
                                            uncond_rows[0] if len(uncond_rows) == 1 else torch.cat(uncond_rows), icond)
            cond_in = cond_rows[0]
            if not uncond_rows:
                return self._forward_region(bbox_id, forward_func, x_tile, sigma_in, original_cond, cond_in, icond)
            uncond_in = uncond_rows[0] if len(uncond_rows) == 1 else torch.cat(uncond_rows)
            if tensor.shape[1] == uncond.shape[1]:
                return self._forward_region(bbox_id, forward_func, x_tile, sigma_in, original_cond,
                                            torch.cat([cond_in, uncond_in]), icond)
            return self._forward_region_split(bbox_id, forward_func, x_tile, sigma_in, original_cond, cond_in, uncond_in, icond, icond)

        # global prompts of different token length: the wrapper runs cond and uncond separately
        if a < T:
            tcond = tensor[a:b]
            if self.is_edit_model:
                tcond = torch.cat([tcond, uncond])
            return self._forward_region(bbox_id, forward_func, x_tile, sigma_in, original_cond, tcond, icond)
        self.set_custom_controlnet_tensors(bbox_id, U)
        self.set_custom_stablesr_tensors(bbox_id)
        return forward_func(x_tile, sigma_in, cond=self.make_cond_dict(original_cond, uncond, icond))

    @custom_bbox
    def ddim_custom_forward(self, x: Tensor, cond_in: CondDict, bbox: CustomBBox, ts: Tensor, forward_func: Callable,
                            *args, **kwargs) -> Tensor:
        """abstractdiffusion.py:429-451: DDIM takes cond and uncond side by side, so only their token counts have
        to agree -- the uncond is padded with its last vector or truncated."""
        tensor, uncond, image_conditioning = self.reconstruct_custom_cond(cond_in, bbox.cond, bbox.uncond, bbox)
        cond = tensor
        if uncond.shape[1] < cond.shape[1]:
            pad = uncond[:, -1:].repeat([1, cond.shape[1] - uncond.shape[1], 1])
            uncond = torch.hstack([uncond, pad])
        elif uncond.shape[1] > cond.shape[1]:
            uncond = uncond[:, :cond.shape[1]]
        if image_conditioning is not None:
            cond = self.make_cond_dict(cond_in, cond, image_conditioning)
            uncond = self.make_cond_dict(cond_in, uncond, image_conditioning)
        return forward_func(x, cond, ts, unconditional_conditioning=uncond, *args, **kwargs)

    _INTERRUPTED = object()

    def _custom_region_pass(self, x: Tensor, custom_func: Callable, poll_interrupt: bool):
        """Second half of a tiled step (multidiffusion.py:170-204, mixtureofdiffusers.py:128-165): every custom region is
        cropped from the latent and denoised by `custom_func`.  The adds into x_buffer / the feather buffers are NOT done
        here: the outputs are collected and composited in one launch by `_composite_regions`.

        Returns [(bbox_id, bbox, x_tile_out)] or `_INTERRUPTED`."""
        done = []
        use_networks = not getattr(self.p, "disable_extra_networks", False)
        for bbox_id, bbox in enumerate(self.custom_bboxes):
            if self._region_skipped(bbox_id):     # inpaint mask: the region lies in the kept area, it and its composite terms drop out
                continue
            if poll_interrupt and host.interrupted():
                return self._INTERRUPTED
            if use_networks:
                host.extra_networks_activate(self.p, bbox.extra_network_data)
            done.append((bbox_id, bbox, custom_func(x[bbox.slicer], bbox_id, bbox)))
            if use_networks:
                host.extra_networks_deactivate(self.p, bbox.extra_network_data)
            self.update_pbar()
        return done

    def _composite_regions(self, x_buffer: Tensor, weights: Optional[Tensor], done, background_aux=None, rows=None, out=None) -> Tensor:
        """x_buffer (grid accumulator) + the collected region outputs -> the step's result, fp32 (td_region_composite:
        BACKGROUND adds in list order, normalisation by `weights` when given, FOREGROUND feather average and overlay).
        rows=(lo, hi): only those canvas rows, written into `out` (td_region_composite_rows, strip shard)."""
        regions = []
        for bbox_id, bbox, r_out in done:
            if bbox.blend_mode == BlendMode.BACKGROUND:
                regions.append((bbox.x, bbox.y, bbox.w, bbox.h, 0, r_out, background_aux(bbox_id) if background_aux is not None else None))
            elif bbox.blend_mode == BlendMode.FOREGROUND:
                regions.append((bbox.x, bbox.y, bbox.w, bbox.h, 1, r_out, bbox.feather_mask))
        w2d = weights.view(x_buffer.shape[2], x_buffer.shape[3]) if weights is not None else None
        if rows is not None:
            return engine.region_composite_rows(x_buffer, w2d, regions, rows[0], rows[1], out)
        return engine.region_composite(x_buffer, w2d, regions)

    # -------------------------------------------------- tiled noise inversion
    @noise_inverse
    def init_noise_inverse(self, steps: int, retouch: float, get_cache_callback, set_cache_callback, renoise_strength: float,
                           renoise_kernel: int):
        """abstractdiffusion.py:591-602: img2img then starts from noise recovered by inverting the input image with the
        tiled denoiser instead of fresh noise; the sampler's `sample_img2img` is replaced for this job."""
        self.noise_inverse_enabled = True
        self.noise_inverse_steps = steps
        self.noise_inverse_retouch = float(retouch)
        self.noise_inverse_renoise_strength = float(renoise_strength)
        self.noise_inverse_renoise_kernel = int(renoise_kernel)
        if self.sample_img2img_original is None:
            self.sample_img2img_original = self.sampler_raw.sample_img2img
        self.sampler_raw.sample_img2img = MethodType(self.sample_img2img, self.sampler_raw)
        self.noise_inverse_set_cache = set_cache_callback
        self.noise_inverse_get_cache = get_cache_callback

    def _renoise_mask(self, p, noise: Tensor) -> Optional[Tensor]:
        """Per-pixel share of fresh noise (abstractdiffusion.py:611-621): 1 - retouch map of the grayscale input,
        bilinearly resized to the latent, times the strength, clamped to [0, 1]."""
        if not self.noise_inverse_renoise_strength > 0:
            return None
        import numpy as np
        import torch.nn.functional as F
        gray = p.init_images[0].convert("L")
        mask = torch.from_numpy(get_retouch_mask(np.asarray(gray), self.noise_inverse_renoise_kernel)).to(noise.device)
        mask = 1 - F.interpolate(mask.unsqueeze(0).unsqueeze(0), size=noise.shape[-2:], mode="bilinear").squeeze(0).squeeze(0)
        mask *= self.noise_inverse_renoise_strength
        return torch.clamp(mask, 0, 1)

    def _cached_inversion(self, p, prompts: List[str], noise: Tensor) -> Optional[Tensor]:
        """The previous run's inverted latent when checkpoint, image, prompts and parameters are unchanged
        (abstractdiffusion.py:625-640)."""
        c = self.noise_inverse_get_cache()
        if c is None:
            return None
        same = (c.model_hash == p.sd_model.sd_model_hash and c.noise_inversion_steps == self.noise_inverse_steps
                and len(c.prompts) == len(prompts) and all(c.prompts[i] == prompts[i] for i in range(len(prompts)))
                and abs(c.retouch - self.noise_inverse_retouch) < 0.01 and c.x0.shape == p.init_latent.shape
                and torch.abs(c.x0.to(p.init_latent.device) - p.init_latent).sum() < 100)
        if not same:
            return None
        print("[Tiled Diffusion] Noise Inversion reuses the cached noise of the previous run (inputs unchanged).")
        return c.xt.to(noise.device)

    def _region_only_noise(self, noise: Tensor) -> Tensor:
        """Without a background layer only the regions are painted: keep the fresh noise under BACKGROUND regions and
        feather it under FOREGROUND regions (abstractdiffusion.py:657-673)."""
        shape = (1, 1, noise.shape[2], noise.shape[3])
        bg_count = torch.zeros(shape, device=noise.device)
        fg_noise = torch.zeros_like(noise)
        fg_weight = torch.zeros(shape, device=noise.device)
        fg_count = torch.zeros(shape, device=noise.device)
        for bbox in self.custom_bboxes:
            if bbox.blend_mode == BlendMode.BACKGROUND:
                bg_count[bbox.slicer] += 1
            elif bbox.blend_mode == BlendMode.FOREGROUND:
                fg_noise[bbox.slicer] += noise[bbox.slicer]
                fg_weight[bbox.slicer] += bbox.feather_mask.to(noise.device)
                fg_count[bbox.slicer] += 1
        bg_noise = torch.where(bg_count > 0, noise, 0)
        fg_noise = torch.where(fg_count > 0, fg_noise / fg_count, 0)
        fg_weight = torch.where(fg_count > 0, fg_weight / fg_count, 0)
        return bg_noise * (1 - fg_weight) + fg_noise * fg_weight

    @noise_inverse
    @keep_signature
    def sample_img2img(self, sampler, p, x: Tensor, noise: Tensor, conditioning, unconditional_conditioning, steps=None,
                       image_conditioning=None):
        """Replacement for `sampler.sample_img2img` (abstractdiffusion.py:604-679): recover (or reuse) the inverted
        latent, turn it into the noise the sampler expects, blend fresh noise back in where the image has detail,
        and hand over to the original img2img sampling."""
        renoise_mask = self._renoise_mask(p, noise)
        prompts = p.all_prompts[:p.batch_size]

        latent = self._cached_inversion(p, prompts, noise)
        if latent is None:
            state = host.get_shared().state
            state.job_count += 1
            latent = self.find_noise_for_image_sigma_adjustment(sampler.model_wrap, self.noise_inverse_steps, prompts)
            state.nextjob()
            self.noise_inverse_set_cache(p.init_latent.clone().cpu(), latent.clone().cpu(), prompts)

        adjusted_steps, _ = host.setup_img2img_steps(p, steps)
        sigmas = sampler.get_sigmas(p, adjusted_steps)
        inverse_noise = latent - (p.init_latent / sigmas[0])

        if renoise_mask is not None:
            if not self.enable_grid_bbox:
                noise = self._region_only_noise(noise)
            combined_noise = ((1 - renoise_mask) * inverse_noise + renoise_mask * noise) / ((renoise_mask ** 2 + (1 - renoise_mask) ** 2) ** 0.5)
        else:
            combined_noise = inverse_noise
        return self.sample_img2img_original(p, x, combined_noise, conditioning, unconditional_conditioning, steps, image_conditioning)

    def _inversion_conditioning(self, prompts: List[str]) -> CondDict:
        """Conditioning of the inversion pass: the job's prompts, no negative prompt, the job's image conditioning."""
        cond = self.p.sd_model.get_learned_conditioning(prompts)
        if isinstance(cond, Tensor):        # SD1 / SD2: one tensor
            return self.make_cond_dict({"c_crossattn": [], "c_concat": []}, cond, self.p.image_conditioning)
        # SDXL: {"crossattn", "vector"}
        return self.make_cond_dict({"crossattn": None, "vector": None, "c_concat": []}, cond["crossattn"], self.p.image_conditioning,
                                   cond["vector"])

    def _inversion_interval(self, dnw, x: Tensor, sigma_from, sigma_to, cond_in: CondDict, step: int, skip: int) -> Tensor:
        """One explicit-Euler interval of the probability-flow ODE dx/dsigma = (x - D(x, sigma)) / sigma, walked UP the
        noise schedule from `sigma_from` to `sigma_to`; D is evaluated at sigma_to with the tiled denoiser, its timestep
        divided by the retouch factor (the img2imgalt "sigma adjustment", abstractdiffusion.py:714-733)."""
        sigma_in = sigma_to * x.new_ones([x.shape[0]])
        c_out, c_in = (k[(...,) + (None,) * (x.ndim - k.ndim)] for k in dnw.get_scalings(sigma_in)[skip:])
        t = dnw.sigma_to_t(sigma_in) / self.noise_inverse_retouch
        eps = self.get_noise(x * c_in, t, cond_in, step)
        denoised = x + eps * c_out
        slope = (x - denoised) / sigma_to
        return x + slope * (sigma_to - sigma_from)

    @noise_inverse
    @torch.no_grad()
    def find_noise_for_image_sigma_adjustment(self, dnw, steps: int, prompts: List[str]) -> Tensor:
        """The latent the sampler would have started from to arrive at the input image (abstractdiffusion.py:681-742):
        integrate the ODE from the image towards noise over the reversed k-diffusion schedule, one tiled denoiser call per
        interval, and return it in units of the largest sigma.  Interruptible between intervals (returns what it has)."""
        assert self.p.sampler_name == "Euler"
        shared = host.get_shared()
        state = shared.state
        skip = 1 if shared.sd_model.parameterization == "v" else 0      # v-models return (c_skip, c_out, c_in)
        schedule = dnw.get_sigmas(steps).flip(0)                         # ascending: 0 -> sigma_max
        cond_in = self._inversion_conditioning(prompts)
        state.sampling_steps = steps
        pbar = None
        if getattr(self.p, "show_tile_progress", True):
            from tqdm import tqdm
            pbar = tqdm(total=steps, desc="Noise Inversion")
        x = self.p.init_latent
        for k in range(1, len(schedule)):
            if state.interrupted:
                return x
            state.sampling_step += 1
            x = self._inversion_interval(dnw, x, schedule[k - 1], schedule[k], cond_in, steps - k, skip)
            host.store_latent(x)
            if pbar is not None:
                pbar.update(1)
        if pbar is not None:
            pbar.close()
        return x / schedule[-1]

    @noise_inverse
    @torch.no_grad()
    def get_noise(self, x_in: Tensor, sigma_in: Tensor, cond_in: CondDict, step: int) -> Tensor:
        raise NotImplementedError

    # ------------------------------------ side-input tile caches (ControlNet, StableSR)
    def _crop_side_input(self, t: Tensor, scale: int, ip: Optional[InpaintPlan] = None) -> Tensor:
        """Every grid tile of a side input [B, C, H*scale, W*scale] in one scatter launch: [T*B, C, th*scale, tw*scale],
        tile-major -- what the reference builds with T slice views and one `cat` per batch (abstractdiffusion.py:494-503).
        With an inpaint plan `ip`: its active tiles only, compact, in tile order."""
        dev = host.device()
        if t.device != dev:
            t = t.to(dev)
        exact = tuple(t.shape[2:]) == (self._grid.H * scale, self._grid.W * scale)
        too_large = max(self._grid.H, self._grid.W) * scale >= 32768
        if self._grid.wrap and (too_large or not exact):
            raise ValueError(f"a wrapped grid crops side inputs modulo the canvas, in the scatter kernel: the input's size "
                             f"{tuple(t.shape[2:])} must be the canvas times {scale}, {(self._grid.H * scale, self._grid.W * scale)}, "
                             "and below 32768")
        if too_large or not exact or not t.is_cuda:
            # beyond the kernels' 16-bit tile origins (a 32k-pixel hint), or a hint whose size is not exactly the scaled
            # canvas (p.width not a multiple of 8, hints resized by the extension: the reference's slicing tolerates
            # both, abstractdiffusion.py:494-503): plain slicing, same tile order
            s = scale
            batches = self.batched_bboxes if ip is None else ip.batched_bboxes
            return torch.cat([t[:, :, b[1] * s:b[3] * s, b[0] * s:b[2] * s] for batch in batches for b in batch], dim=0)
        if ip is not None:
            origins = ip.origins_dev * scale
            host_origins = (ctypes.c_int32 * len(ip.origins_host))(*[v * scale for v in ip.origins_host])
            return engine.scatter_bboxes(t.contiguous(), origins, host_origins, ip.num_tiles, self._grid.tile_h * scale,
                                         self._grid.tile_w * scale)
        g = self._grid if scale == 1 else engine.scaled_grid(self._grid, scale)
        return engine.scatter_tiles(g, t.contiguous(), flags=self._blend_flags)

    def _batch_rows(self, tiles: Tensor, batch_id: int, rows_per_tile: int, num_tiles: Optional[int] = None) -> Tensor:
        lo = batch_id * self.tile_bs * rows_per_tile
        hi = min((batch_id + 1) * self.tile_bs, self.num_tiles if num_tiles is None else num_tiles) * rows_per_tile
        return tiles[lo:hi]

    def _side_input_tiles(self, full: Tensor, scale: int, park_on_cpu: bool):
        """(per tile batch, per custom region) crops of one side input living at `scale` x the latent resolution."""
        park = (lambda t: t.cpu()) if park_on_cpu else (lambda t: t)
        per_batch, per_region = [], []
        ip = self._inpaint
        if ip is not None and self.batched_bboxes:      # inpaint mask: the active tiles only, in the compact batches of the loop
            if ip.batched_bboxes:
                tiles = self._crop_side_input(full, scale, ip)
                per_batch = [park(self._batch_rows(tiles, b, full.shape[0], ip.num_tiles)) for b in range(len(ip.batched_bboxes))]
        elif self.batched_bboxes:
            tiles = self._crop_side_input(full, scale)
            rows = full.shape[0]
            per_batch = [park(self._batch_rows(tiles, b, rows)) for b in range(len(self.batched_bboxes))]
        for bbox in self.custom_bboxes:
            per_region.append(park(full[:, :, bbox[1] * scale:bbox[3] * scale, bbox[0] * scale:bbox[2] * scale]))
        return per_batch, per_region

    @controlnet
    def init_controlnet(self, controlnet_script, control_tensor_cpu: bool):
        """Register the ControlNet extension's script object; its hints are cropped once per job
        (abstractdiffusion.py:454-464)."""
        self.enable_controlnet = True
        self.controlnet_script = controlnet_script
        self.control_tensor_cpu = control_tensor_cpu
        self.control_tensor_batch = None
        self.control_params = None
        self.control_tensor_custom = []
        self.prepare_controlnet_tensors()

    def _control_params(self):
        return self.control_params if (self.enable_controlnet and self.control_tensor_batch is not None) else []

    @controlnet
    def reset_controlnet_tensors(self):
        """Hand every ControlNet unit its full-size hint back (abstractdiffusion.py:466-472)."""
        for unit, full in zip(self._control_params(), getattr(self, "org_control_tensor_batch", [])):
            unit.hint_cond = full

    @controlnet
    def prepare_controlnet_tensors(self, refresh: bool = False):
        """Crop the hint of every ControlNet unit into the tile batches and the custom regions, once per job
        (abstractdiffusion.py:474-518).  Hints live in pixel space, i.e. at opt_f x the latent grid; all grid tiles of
        one hint come from ONE scatter launch and `control_tensor_batch[unit][batch]` are views of its output."""
        if not refresh and (self.control_tensor_batch is not None or self.control_params is not None):
            return
        if not self.enable_controlnet or self.controlnet_script is None:
            return
        network = self.controlnet_script.latest_network
        if network is None or not hasattr(network, "control_params"):
            return
        self.control_params = network.control_params
        self.org_control_tensor_batch = [unit.hint_cond for unit in self.control_params]
        if not self.org_control_tensor_batch:
            return
        self.control_tensor_batch, self.control_tensor_custom = [], []      # (the reference keeps stale region crops on refresh)
        for hint in self.org_control_tensor_batch:
            if hint.dim() == 3:
                hint.unsqueeze_(0)          # in place, like the reference: the unit sees a 4-d hint from now on
            per_batch, per_region = self._side_input_tiles(hint, opt_f, self.control_tensor_cpu)
            self.control_tensor_batch.append(per_batch)
            if per_region:
                self.control_tensor_custom.append(per_region)

    @controlnet
    def switch_controlnet_tensors(self, batch_id: int, x_batch_size: int, tile_batch_size: int, is_denoise=False):
        """Point every ControlNet unit at the hint crops of tile batch `batch_id`, replicated the way the sampler
        replicates the latent (abstractdiffusion.py:520-535): k-diffusion keeps the x_batch_size copies of a tile
        adjacent, the DDIM family repeats the whole tile batch (twice more when cond and uncond run together)."""
        for unit_id, unit in enumerate(self._control_params()):
            crops = self._side_batch(self.control_tensor_batch[unit_id], self.org_control_tensor_batch[unit_id], opt_f, batch_id)
            if self.is_kdiff:
                crops = crops[:tile_batch_size].repeat_interleave(x_batch_size, dim=0)
            else:
                crops = crops.repeat([x_batch_size * (1 if is_denoise else 2), 1, 1, 1])
            unit.hint_cond = crops.to(host.device())

    def _side_batch(self, per_batch: list, full: Tensor, scale: int, batch_id: int) -> Tensor:
        """A side input's crops for tile batch `batch_id` of the loop that runs.  The caches hold the inpaint plan's active tiles;
        the full-plan pass of noise inversion crops its batch from the whole side input instead."""
        if self._inpaint is None or not self._full_plan_pass:
            return per_batch[batch_id]
        bboxes = self.batched_bboxes[batch_id]
        s = scale
        return torch.cat([full[:, :, b.y * s:(b.y + b.h) * s, b.x * s:(b.x + b.w) * s] for b in bboxes], dim=0)

    @controlnet
    def set_custom_controlnet_tensors(self, bbox_id: int, repeat_size: int):
        """The hint crop of custom region `bbox_id`, once per latent in the region's batch (abstractdiffusion.py:537-544)."""
        if not self.enable_controlnet or not len(self.control_tensor_custom):
            return
        for unit_id, unit in enumerate(self.control_params):
            unit.hint_cond = self.control_tensor_custom[unit_id][bbox_id].to(host.device()).repeat((repeat_size, 1, 1, 1))

    def _stablesr_model(self):
        script = getattr(self, "stablesr_script", None)
        model = getattr(script, "stablesr_model", None) if script is not None else None
        return model if self.enable_stablesr else None

    @stablesr
    def init_stablesr(self, stablesr_script):
        """StableSR publishes its conditioning latent through a hook (abstractdiffusion.py:547-568); when it does, crop
        it into the tile batches and regions (latent space: the grid as is, one scatter launch)."""
        if stablesr_script.stablesr_model is None:
            return
        self.stablesr_script = stablesr_script

        def on_latent_image(latent_image):
            self.enable_stablesr = True
            self.stablesr_tensor = latent_image
            per_batch, per_region = self._side_input_tiles(latent_image, 1, False)
            self.stablesr_tensor_batch = per_batch
            if per_region:
                self.stablesr_tensor_custom = per_region

        stablesr_script.stablesr_model.set_image_hooks["TiledDiffusion"] = on_latent_image

    @stablesr
    def reset_stablesr_tensors(self):
        model = self._stablesr_model()
        if model is not None:
            model.latent_image = self.stablesr_tensor

    @stablesr
    def switch_stablesr_tensors(self, batch_id: int):
        model = self._stablesr_model()
        if model is not None and self.stablesr_tensor_batch is not None:
            model.latent_image = self._side_batch(self.stablesr_tensor_batch, self.stablesr_tensor, 1, batch_id)

    @stablesr
    def set_custom_stablesr_tensors(self, bbox_id: int):
        model = self._stablesr_model()
        crops = getattr(self, "stablesr_tensor_custom", [])
        if model is not None and len(crops):
            model.latent_image = crops[bbox_id]

    # ----------------------------------------------------------- engine glue
    def _check_input(self, x_in: Tensor) -> Tensor:
        if not x_in.is_cuda:
            raise RuntimeError(f"{self.method}: latent is on {x_in.device}; the H100 path has no CPU fallback")
        if self.enable_grid_bbox and self._grid is None:
            raise RuntimeError(f"{self.method}: init_grid_bbox() has not been called")
        if self.weights.device != x_in.device:
            self.weights = self.weights.to(x_in.device)
        if self._rcp_weights is not None and self._rcp_weights.device != x_in.device:
            self._rcp_weights = self._rcp_weights.to(x_in.device)
        return x_in.contiguous()

    def _scatter_all(self, x_in: Tensor) -> Tensor:
        """One launch: every grid tile of this step, tile-major (multidiffusion.py:155 for all batches)."""
        self._tiles = engine.scatter_tiles(self._grid, x_in, out=self._tiles, flags=self._blend_flags)
        return self._tiles

    def _tile_batch(self, tiles: Tensor, batch_id: int, N: int) -> Tensor:
        lo = batch_id * self.tile_bs * N
        hi = min((batch_id + 1) * self.tile_bs, self.num_tiles) * N
        return tiles[lo:hi]

    def cat_repeat(self, x: Tensor, n: int) -> Tensor:
        """`torch.cat([x] * n, dim=0)` (mixtureofdiffusers.py:91-99), memoised per source tensor object and version: the
        batches of one UNet call repeat the same timestep / cond tensors, one copy serves them all."""
        if n == 1:
            return x
        cache = self.__dict__.setdefault("_cat_cache", {})
        key = (id(x), n)
        hit = cache.get(key)
        if hit is not None and hit[0] is x and hit[1] == x._version:
            return hit[2]
        out = torch.cat([x] * n, dim=0)
        if len(cache) > 16:
            cache.clear()
        cache[key] = (x, x._version, out)   # the strong reference keeps id(x) from being recycled
        return out

    def _tile_batch_views(self, tiles: Tensor, N: int) -> List[Tensor]:
        """The per-batch views of the persistent tile buffer, built once per buffer (not once per sampler step)."""
        cached = self.__dict__.get("_tile_views_cache")
        if cached is not None and cached[0] is tiles and cached[1] == N:
            return cached[2]
        views = [self._tile_batch(tiles, b, N) for b in range(self.num_batches)]
        self._tile_views_cache = (tiles, N, views)
        return views

    def _icond_tile_batches(self, icond: Tensor):
        """img2img: spatial icond is cropped per tile like the latent (multidiffusion.py:121-122)."""
        self._icond_tiles = engine.scatter_tiles(self._grid, icond, out=self._icond_tiles, flags=self._blend_flags)
        return self._icond_tiles

    def repeat_tensor(self, x: Tensor, n: int) -> Tensor:
        """Repeat on dim 0 (multidiffusion.py:100-110): expand when B == 1, else tile.

        The tiled copy is memoised per source tensor OBJECT (+ version): all T/tile_bs batches of a step
        repeat the same cond, so the reference's per-batch `repeat` becomes one launch per step."""
        if n == 1:
            return x
        r_dims = x.dim() - 1
        if x.shape[0] == 1:
            return x.expand([n] + [-1] * r_dims)
        cache = self.__dict__.setdefault("_repeat_cache", {})
        key = (id(x), n)
        hit = cache.get(key)
        if hit is not None and hit[0] is x and hit[1] == x._version:
            return hit[2]
        out = x.repeat([n] + [1] * r_dims)
        if len(cache) > 16:
            cache.clear()
        cache[key] = (x, x._version, out)   # the strong reference keeps id(x) from being recycled
        return out
