"""MultiDiffusion (arXiv 2302.08113) tile method with the reference's surface
(tile_methods/multidiffusion.py), executed by two sm_90a kernels per sampler step:

    td_scatter_tiles          <- `torch.cat([x_in[bbox.slicer] ...])` for every batch   (:155)
    td_blend_multidiffusion   <- `x_buffer[slicer] += tile` x T  +  `torch.where(...)`   (:166-167, :208)

The UNet (`repeat_func`) stays the host application's; it receives views of the
persistent tile buffer and its output tensors are read in place by the blend
kernel (pointer table, no concatenation copy).
"""
from __future__ import annotations

import ctypes
from typing import Callable, List, Optional, Union

import torch
from torch import Tensor

from .. import engine, host
from ..tile_utils.utils import BBox, BlendMode, CustomBBox, custom_bbox, keep_signature
from .abstractdiffusion import AbstractDiffusion, CondDict


class MultiDiffusion(AbstractDiffusion):

    def __init__(self, p, *args, **kwargs):
        super().__init__(p, *args, **kwargs)
        assert p.sampler_name != "UniPC", "MultiDiffusion is not compatible with UniPC!"

    # ---------------------------------------------------------------- hooks
    def hook(self):
        """Patch `sampler.model_wrap_cfg.inner_model.forward` (multidiffusion.py:15-29)."""
        inner = self.sampler.model_wrap_cfg.inner_model
        self.sampler_forward = inner.forward
        inner.forward = self.kdiff_forward if self.is_kdiff else self.ddim_forward

    @staticmethod
    def unhook():
        # the patched sampler object dies with the generation job (multidiffusion.py:31-35)
        pass

    def reset_buffer(self, x_in: Tensor):
        super().reset_buffer(x_in)

    @custom_bbox
    def init_custom_bbox(self, *args):
        """multidiffusion.py:40-46: a BACKGROUND region counts as one more tile in the weight canvas."""
        super().init_custom_bbox(*args)
        for bbox in self.custom_bboxes:
            if bbox.blend_mode == BlendMode.BACKGROUND:
                self.weights[bbox.slicer] += 1.0

    # ------------------------------------------------------- kernel hijacks
    @torch.no_grad()
    @keep_signature
    def kdiff_forward(self, x_in: Tensor, sigma_in: Tensor, cond: CondDict) -> Tensor:
        def org_func(x: Tensor) -> Tensor:
            return self.sampler_forward(x, sigma_in, cond=cond)

        def repeat_func(x_tile: Tensor, bboxes: List[BBox]) -> Tensor:
            sigma_tile = self.repeat_tensor(sigma_in, len(bboxes))
            cond_tile = self.repeat_cond_dict(cond, bboxes)
            return self.sampler_forward(x_tile, sigma_tile, cond=cond_tile)

        def custom_func(x: Tensor, bbox_id: int, bbox: CustomBBox) -> Tensor:
            return self.kdiff_custom_forward(x, sigma_in, cond, bbox_id, bbox, self.sampler_forward)

        return self.sample_one_step(x_in, org_func, repeat_func, custom_func)

    @torch.no_grad()
    @keep_signature
    def ddim_forward(self, x_in: Tensor, ts_in: Tensor, cond: Union[CondDict, Tensor]) -> Tensor:
        def org_func(x: Tensor) -> Tensor:
            return self.sampler_forward(x, ts_in, cond=cond)

        def repeat_func(x_tile: Tensor, bboxes: List[BBox]) -> Tensor:
            n_rep = len(bboxes)
            ts_tile = self.repeat_tensor(ts_in, n_rep)
            if isinstance(cond, dict):
                cond_tile = self.repeat_cond_dict(cond, bboxes)
            else:
                cond_tile = self.repeat_tensor(cond, n_rep)
            return self.sampler_forward(x_tile, ts_tile, cond=cond_tile)

        def custom_func(x: Tensor, bbox_id: int, bbox: CustomBBox) -> Tensor:
            def forward_func(x, *args, **kwargs):
                self.set_custom_controlnet_tensors(bbox_id, 2 * x.shape[0])
                self.set_custom_stablesr_tensors(bbox_id)
                return self.sampler_forward(x, *args, **kwargs)
            return self.ddim_custom_forward(x, cond, bbox, ts_in, forward_func)

        return self.sample_one_step(x_in, org_func, repeat_func, custom_func)

    def repeat_cond_dict(self, cond_in: CondDict, bboxes: List[BBox]) -> CondDict:
        """Per-batch cond (multidiffusion.py:112-129): text/vector cond repeated, spatial icond cropped per tile.

        Without a spatial icond the result only depends on (cond_in, len(bboxes)): every batch of a step gets a shallow
        copy of one memoised dict instead of rebuilding it (the tensors inside are shared, as they are read-only)."""
        n_rep = len(bboxes)
        memo = self.__dict__.get("_cond_memo")
        token = self.__dict__.get("_step_token", 0)
        if memo is not None and memo[0] is cond_in and memo[1] == n_rep:
            if memo[5] == token:                       # validated earlier in this sampler step
                return dict(memo[3])
            if memo[2] == self._cond_versions(cond_in):
                self._cond_memo = memo[:5] + (token,)
                return dict(memo[3])
        tcond = self.repeat_tensor(self.get_tcond(cond_in), n_rep)
        icond = self.get_icond(cond_in)
        spatial = tuple(icond.shape[2:]) == (self.h, self.w)
        if spatial:
            icond = self._crop_icond(icond, bboxes)
        else:
            icond = self.repeat_tensor(icond, n_rep)
        vcond = self.get_vcond(cond_in)
        if vcond is not None:
            vcond = self.repeat_tensor(vcond, n_rep)
        out = self.make_cond_dict(cond_in, tcond, icond, vcond)
        if not spatial:
            # the source tensors are kept alive with the memo so that their ids cannot be recycled
            sources = (self.get_tcond(cond_in), self.get_icond(cond_in), self.get_vcond(cond_in))
            self._cond_memo = (cond_in, n_rep, self._cond_versions(cond_in), out, sources, token)
            return dict(out)
        return out

    def _cond_versions(self, cond_in: CondDict):
        """Identity + in-place version of the tensors a memoised cond dict was built from."""
        t, i, v = self.get_tcond(cond_in), self.get_icond(cond_in), self.get_vcond(cond_in)
        return (id(t), t._version, id(i), i._version, None if v is None else (id(v), v._version))

    def _crop_icond(self, icond: Tensor, bboxes: List[BBox]) -> Tensor:
        """Spatial icond -> tile batch with the same scatter kernel as the latent (a batch of the inpaint plan's active tiles need
        not be a contiguous tile range: its windows go through the list scatter)."""
        if self._active_plan() is not None:
            flat = [v for b in bboxes for v in (b.x, b.y)]
            return engine.scatter_bboxes(icond.contiguous(), torch.tensor(flat, dtype=torch.int32, device=icond.device),
                                         (ctypes.c_int32 * len(flat))(*flat), len(bboxes), self.tile_h, self.tile_w)
        first = self._bbox_index(bboxes[0])
        return engine.scatter_tiles(self._grid, icond, tile_begin=first, tile_end=first + len(bboxes),
                                    flags=self._blend_flags)

    def _bbox_index(self, bbox: BBox) -> int:
        g = self._grid
        r = list(g.ys[:g.rows]).index(bbox.y)
        c = list(g.xs[:g.cols]).index(bbox.x)
        return r * g.cols + c

    def sample_one_step(self, x_in: Tensor, org_func: Callable, repeat_func: Callable, custom_func: Callable) -> Tensor:
        """One denoiser call over the whole latent, tile by tile, then region by region (multidiffusion.py:131-218).

        Returns a fresh fp32 tensor, as the reference's `torch.where` against the
        fp32 weights does even for fp16 latents.
        """
        N, C, H, W = x_in.shape
        if (H, W) != (self.h, self.w):
            # hires-fix second pass is not tiled (multidiffusion.py:141-144)
            self.reset_controlnet_tensors()
            return org_func(x_in)

        x = self._check_input(x_in)
        self._step_token = self.__dict__.get("_step_token", 0) + 1     # memoised per-batch inputs are re-validated once per step
        regions = self.enable_custom_bbox and len(self.custom_bboxes) > 0
        if self._shard is not None:
            return self._sample_one_step_sharded(x_in, x, repeat_func, custom_func if regions else None, N, C)

        x_out = None
        ip = self._active_plan()
        if self.enable_grid_bbox and ip is not None:
            # inpaint mask: the active tiles only, in compact batches; the sparse blend drops the skipped tiles' visits
            outs = []
            tiles = self._scatter_active(x, ip) if ip.num_tiles else None
            side_inputs = self.enable_controlnet or self.enable_stablesr
            off = 0
            for batch_id, bboxes in enumerate(ip.batched_bboxes):
                if host.interrupted():
                    return x_in
                if side_inputs:
                    self.switch_controlnet_tensors(batch_id, N, len(bboxes))
                    self.switch_stablesr_tensors(batch_id)
                outs.append(repeat_func(tiles[off * N:(off + len(bboxes)) * N], bboxes))
                off += len(bboxes)
                if self.pbar is not None:
                    self.update_pbar()
            if regions:
                self.reset_buffer(x)
            x_out = engine.blend_multidiffusion_sparse(self._grid, outs, N, C, self.tile_bs, self.weights, x.dtype, ip.slot_dev, ip.slot_host,
                                                       x_buffer=self.x_buffer if regions else None, flags=self._blend_flags,
                                                       rcp_weights=self._rcp_weights, tile_dtype=x.dtype)
            if not regions:
                return x_out
        elif self.enable_grid_bbox:
            tiles = self._scatter_all(x)
            views = self._tile_batch_views(tiles, N)
            state = getattr(host.get_shared(), "state", None)      # polled per tile batch (multidiffusion.py:152)
            side_inputs = self.enable_controlnet or self.enable_stablesr
            outs = []
            for batch_id, bboxes in enumerate(self.batched_bboxes):
                if state is not None and getattr(state, "interrupted", False):
                    return x_in
                if side_inputs:
                    self.switch_controlnet_tensors(batch_id, N, len(bboxes))
                    self.switch_stablesr_tensors(batch_id)
                outs.append(repeat_func(views[batch_id], bboxes))
                if self.pbar is not None:
                    self.update_pbar()
            if regions:
                self.reset_buffer(x)        # the regions composite on top of the UN-normalised accumulator
            x_out = engine.blend_multidiffusion(self._grid, outs, N, C, self.tile_bs, self.weights, x.dtype,
                                                x_buffer=self.x_buffer if regions else None, flags=self._blend_flags,
                                                rcp_weights=self._rcp_weights)
            if not regions:
                return x_out
        else:
            # draw_background=False: only the custom regions paint (multidiffusion.py:146 skips the grid loop)
            self.reset_buffer(x)
            self.x_buffer.zero_()

        done = self._custom_region_pass(x, custom_func, poll_interrupt=True)
        if done is self._INTERRUPTED:
            return x_in
        # multidiffusion.py:187-216 in one launch: BACKGROUND adds, divide where weights > 1, FOREGROUND feather overlay
        return self._composite_regions(self.x_buffer, self.weights, done)

    def _sample_one_step_sharded(self, x_in: Tensor, x: Tensor, repeat_func: Callable, custom_func: Optional[Callable], N: int,
                                 C: int) -> Tensor:
        """This rank's tiles (and custom regions, when `custom_func` is given), then the exchange + deterministic blend
        (init_tile_shard), then the region composite over the blend's accumulator.

        An interrupt (multidiffusion.py:152) stops the denoiser calls of THIS rank but not its part of the exchange:
        the peers' kernels wait for this rank's signal, so the step always publishes (possibly stale) tile outputs,
        blends and signals -- the step counters stay in lock-step -- and only then returns x_in like the reference."""
        sh = self._shard
        outs = []
        interrupted = False
        if self.enable_grid_bbox and sh.num_local > 0:
            self._tiles = engine.scatter_tiles(self._grid, x, out=self._tiles, tile_begin=sh.begin, tile_end=sh.end,
                                               flags=self._blend_flags)
            off = 0
            for batch_id, bboxes in enumerate(self.local_batched_bboxes):
                x_tile = self._tiles[off * N:(off + len(bboxes)) * N]
                off += len(bboxes)
                if interrupted or host.interrupted():
                    interrupted = True
                    outs.append(x_tile)          # placeholder with the right shape: the exchange must still happen
                    continue
                outs.append(repeat_func(x_tile, bboxes))
                self.update_pbar()
        done = None
        if custom_func is not None:
            # the region exchange (NCCL) comes before the tile exchange: its in-kernel waits then never sit in front of a collective
            self.reset_buffer(x)
            done, interrupted = self._region_pass_sharded(x, custom_func, True, interrupted)
        if self._shard_mode == "strip":
            out = self._strip_step(outs, x, N, C, done)
        elif done is None:
            out = self._exchange_and_blend_md(outs, x, N, C)
        else:
            if self.enable_grid_bbox:
                self._exchange_and_blend_md(outs, x, N, C, x_buffer=self.x_buffer)
            else:
                self.x_buffer.zero_()
            out = self._composite_regions(self.x_buffer, self.weights, done)
        return x_in if interrupted else out

    def _strip_latent_dtype(self, x_dtype: torch.dtype) -> torch.dtype:
        return torch.float32            # the normalising divide (multidiffusion.py:208) is fp32

    def _strip_blend(self, ex, x: Tensor, x_buffer: Optional[Tensor]):
        ex.blend(self._grid, self.weights, self._rcp_weights if x.dtype != torch.float32 else None, flags=self._blend_flags, x_buffer=x_buffer)

    def _region_composite_terms(self):
        return self.weights, None

    def get_noise(self, x_in: Tensor, sigma_in: Tensor, cond_in: CondDict, step: int) -> Tensor:
        """Tiled eps prediction used by noise inversion (multidiffusion.py:220-243)."""
        from ..tile_utils.utils import Condition
        cond_orig = cond_in.copy()
        sd_model = self._sd_model()

        def org_func(x: Tensor):
            return sd_model.apply_model(x, sigma_in, cond=cond_orig)

        def repeat_func(x_tile: Tensor, bboxes: List[BBox]):
            sigma_tile = sigma_in.repeat(len(bboxes))
            cond_out = self.repeat_cond_dict(cond_orig, bboxes)
            return sd_model.apply_model(x_tile, sigma_tile, cond=cond_out)

        def custom_func(x: Tensor, bbox_id: int, bbox: CustomBBox):
            # the region's negative prompt is deliberately not used for noise inversion (multidiffusion.py:233-235)
            tcond = Condition.reconstruct_cond(bbox.cond, step).unsqueeze_(0)
            icond = self.get_icond(cond_orig)
            if tuple(icond.shape[2:]) == (self.h, self.w):
                icond = icond[bbox.slicer]
            return sd_model.apply_model(x, sigma_in, cond=self.make_cond_dict(cond_in, tcond, icond))

        # the inverted latent is the full plan's: there is no host mask here, and an active tile reads kept pixels too
        self._full_plan_pass = True
        try:
            return self.sample_one_step(x_in, org_func, repeat_func, custom_func)
        finally:
            self._full_plan_pass = False
