"""Mixture of Diffusers tile method with the reference's surface
(tile_methods/mixtureofdiffusers.py): hooks `sd_model.apply_model`, fuses the
per-tile eps with gaussian weights that are pre-normalised by 1/sum(weights).

Per UNet call: td_scatter_tiles + td_blend_mixture (the reference: T/TB cats and
3T elementwise kernels).  The blend reproduces `w = tile_weights *
rescale_factor[slicer]; x_buffer[slicer] += eps * w` with the same separate
roundings, so results are bit-identical to the reference.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import Tensor

from .. import engine, host
from ..tile_utils.utils import BBox, BlendMode, Condition, CustomBBox, custom_bbox, gaussian_weights, grid_bbox, keep_signature
from .abstractdiffusion import AbstractDiffusion, CondDict

_STRIP_NO_INVERSION = "the row-strip shard of Mixture of Diffusers does not run tiled noise inversion: use mode='replicate'"


class MixtureOfDiffusers(AbstractDiffusion):

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.custom_weights: List[Tensor] = []
        self.get_weight = gaussian_weights

    def hook(self):
        """mixtureofdiffusers.py:18-21."""
        sd_model = self._sd_model()
        if not hasattr(sd_model, "apply_model_original_md"):
            sd_model.apply_model_original_md = sd_model.apply_model
        sd_model.apply_model = self.apply_model_hijack
        self._hooked_model = sd_model

    @staticmethod
    def unhook():
        """mixtureofdiffusers.py:23-27."""
        sd_model = getattr(host.get_shared(), "sd_model", None)
        if sd_model is not None and hasattr(sd_model, "apply_model_original_md"):
            sd_model.apply_model = sd_model.apply_model_original_md
            del sd_model.apply_model_original_md

    def init_done(self):
        """mixtureofdiffusers.py:29-36: rescale_factor = 1 / weights, once, in fp32."""
        super().init_done()
        w_host = self.weights.detach().to("cpu", torch.float32).numpy().reshape(self.h, self.w)
        rf = engine.rescale_factor(w_host)
        self.rescale_factor = torch.from_numpy(rf).view(1, 1, self.h, self.w).to(self.weights.device)
        # BACKGROUND regions: their gaussians are pre-multiplied by the rescale factor once (mixtureofdiffusers.py:33-36)
        for bbox_id, bbox in enumerate(self.custom_bboxes):
            if bbox.blend_mode == BlendMode.BACKGROUND:
                self.custom_weights[bbox_id] *= self.rescale_factor[bbox.slicer]

    @grid_bbox
    def get_tile_weights(self) -> Tensor:
        """mixtureofdiffusers.py:38-43."""
        if not hasattr(self, "tile_weights"):
            self.tile_weights = self.get_weight(self.tile_w, self.tile_h)
        return self.tile_weights

    @custom_bbox
    def init_custom_bbox(self, *args):
        """mixtureofdiffusers.py:45-55: a BACKGROUND region brings its own gaussian (sized to the region) into the
        weight canvas; `init_done` then rescales it like the grid tiles' gaussian."""
        super().init_custom_bbox(*args)
        self.custom_weights = []
        for bbox in self.custom_bboxes:
            if bbox.blend_mode == BlendMode.BACKGROUND:
                cw = self.get_weight(bbox.w, bbox.h).to(self.weights.device)
                self.weights[bbox.slicer] += cw
                self.custom_weights.append(cw.clone().unsqueeze(0).unsqueeze(0))
            else:
                self.custom_weights.append(None)

    @torch.no_grad()
    @keep_signature
    def apply_model_hijack(self, x_in: Tensor, t_in: Tensor, cond: CondDict, noise_inverse_step: int = -1):
        """mixtureofdiffusers.py:61-179.  Returns `x_buffer` (aliases delegate state, like the reference) unless
        FOREGROUND regions were composited over it."""
        sd_model = self._sd_model()
        c_in: CondDict = cond
        N, C, H, W = x_in.shape
        if (H, W) != (self.h, self.w):
            self.reset_controlnet_tensors()
            return sd_model.apply_model_original_md(x_in, t_in, c_in)

        x = self._check_input(x_in)
        self.reset_buffer(x)
        regions = self.enable_custom_bbox and len(self.custom_bboxes) > 0

        def custom_func(x_tile: Tensor, bbox_id: int, bbox: CustomBBox) -> Tensor:
            if noise_inverse_step < 0:
                return self.custom_apply_model(x_tile, t_in, c_in, bbox_id, bbox)
            tcond = Condition.reconstruct_cond(bbox.cond, noise_inverse_step)
            icond = self.get_icond(c_in)
            if tuple(icond.shape[2:]) == (self.h, self.w):
                icond = icond[bbox.slicer]
            c_out = self.make_cond_dict(c_in, tcond, icond, self.get_vcond(c_in))
            return sd_model.apply_model(x_tile, t_in, cond=c_out)

        if self._strip is not None:
            if noise_inverse_step >= 0:
                raise NotImplementedError(_STRIP_NO_INVERSION)
            return self._apply_strip(x_in, x, t_in, c_in, sd_model, N, C, custom_func if regions else None)
        interrupted = False

        if self.enable_grid_bbox:
            x_out = self._grid_pass(x_in, x, t_in, c_in, sd_model, N, C)
            if x_out is None:
                if self._shard is None or not regions:
                    return x_in        # interrupted
                interrupted = True     # sharded: the region exchange still has to happen
        else:
            # draw_background=False: only the custom regions paint (mixtureofdiffusers.py:82 skips the grid loop)
            self.x_buffer.zero_()
        if not regions:
            return self.x_buffer

        if self._shard is not None:
            done, interrupted = self._region_pass_sharded(x, custom_func, False, interrupted)
            if interrupted:
                return x_in
        else:
            done = self._custom_region_pass(x, custom_func, poll_interrupt=False)
        # mixtureofdiffusers.py:145-175 in one launch: BACKGROUND adds weighted by the pre-rescaled custom weights, no
        # normalisation, FOREGROUND feather overlay
        out = self._composite_regions(self.x_buffer, None, done, background_aux=lambda bbox_id: self.custom_weights[bbox_id])
        if any(b.blend_mode == BlendMode.FOREGROUND for b in self.custom_bboxes):
            return out                       # the reference's overlay promotes to fp32 (fp32 mask; so also when the inpaint mask skips it)
        self.x_buffer.copy_(out)             # BACKGROUND only: the reference returns x_buffer itself (x_in.dtype; lossless)
        return self.x_buffer

    def _denoise_tile_batch(self, sd_model, x_tile: Tensor, n_rep: int, t_in: Tensor, c_in: CondDict, icond_tile, batch_id: int,
                            N: int) -> Tensor:
        """One UNet call on a batch of n_rep tiles: timestep / text / vector cond repeated per tile, spatial image cond
        already cropped per tile (mixtureofdiffusers.py:89-119)."""
        t_tile = self.cat_repeat(t_in, n_rep)
        if not isinstance(c_in, dict):
            raise NotImplementedError("non-dict conditioning is not supported by Mixture of Diffusers "
                                      "(the reference only prints a warning here, mixtureofdiffusers.py:103)")
        tcond_tile = self.cat_repeat(self.get_tcond(c_in), n_rep)
        if icond_tile is None:
            icond_tile = self.cat_repeat(self.get_icond(c_in), n_rep)
        vcond = self.get_vcond(c_in)
        vcond_tile = None if vcond is None else self.cat_repeat(vcond, n_rep)
        c_tile = self.make_cond_dict(c_in, tcond_tile, icond_tile, vcond_tile)
        self.switch_controlnet_tensors(batch_id, N, n_rep, is_denoise=True)
        self.switch_stablesr_tensors(batch_id)
        return sd_model.apply_model_original_md(x_tile, t_tile, c_tile)

    def _grid_pass(self, x_in: Tensor, x: Tensor, t_in: Tensor, c_in: CondDict, sd_model, N: int, C: int):
        """Grid tiles of one UNet call: scatter, denoise per batch, fused gaussian blend into x_buffer.
        Returns x_buffer, or None when the job was interrupted."""
        self._blend_inputs_to(x.device)
        if self._shard is not None:
            return self._grid_pass_sharded(x, t_in, c_in, sd_model, N, C)

        ip = self._active_plan()
        if ip is not None:
            return self._grid_pass_active(ip, x, t_in, c_in, sd_model, N, C)
        tiles = self._scatter_all(x)
        icond_tiles = None
        if isinstance(c_in, dict):
            icond_full = self.get_icond(c_in)
            if tuple(icond_full.shape[2:]) == (self.h, self.w):
                icond_tiles = self._icond_tile_batches(icond_full)
                n_icond = icond_full.shape[0]

        outs = []
        for batch_id, bboxes in enumerate(self.batched_bboxes):
            if host.interrupted():
                return None
            n_rep = len(bboxes)
            x_tile = self._tile_batch(tiles, batch_id, N)
            icond_tile = self._tile_batch(icond_tiles, batch_id, n_icond) if icond_tiles is not None else None
            outs.append(self._denoise_tile_batch(sd_model, x_tile, n_rep, t_in, c_in, icond_tile, batch_id, N))
            self.update_pbar()

        return engine.blend_mixture(self._grid, outs, N, C, self.tile_bs, self.tile_weights, self.rescale_factor,
                                    self.x_buffer, flags=self._blend_flags)

    def _grid_pass_active(self, ip, x: Tensor, t_in: Tensor, c_in: CondDict, sd_model, N: int, C: int):
        """`_grid_pass` under an inpaint mask: the active tiles in compact batches (latent and spatial image cond through the list
        scatter), then the sparse gaussian blend, which drops the skipped tiles' visits.  Returns x_buffer, or None when
        interrupted."""
        outs = []
        if ip.num_tiles:
            tiles = self._scatter_active(x, ip)
            icond_tiles, n_icond = None, 0
            if isinstance(c_in, dict):
                icond_full = self.get_icond(c_in)
                if tuple(icond_full.shape[2:]) == (self.h, self.w):
                    icond_tiles = engine.scatter_bboxes(icond_full.contiguous(), ip.origins_dev, ip.origins_host, ip.num_tiles,
                                                        self.tile_h, self.tile_w)
                    n_icond = icond_full.shape[0]
            off = 0
            for batch_id, bboxes in enumerate(ip.batched_bboxes):
                if host.interrupted():
                    return None
                n_rep = len(bboxes)
                icond_tile = icond_tiles[off * n_icond:(off + n_rep) * n_icond] if icond_tiles is not None else None
                outs.append(self._denoise_tile_batch(sd_model, tiles[off * N:(off + n_rep) * N], n_rep, t_in, c_in, icond_tile, batch_id, N))
                off += n_rep
                self.update_pbar()
        return engine.blend_mixture_sparse(self._grid, outs, N, C, self.tile_bs, self.tile_weights, self.rescale_factor, self.x_buffer,
                                           ip.slot_dev, ip.slot_host, flags=self._blend_flags, tile_dtype=x.dtype)

    def _blend_inputs_to(self, device):
        if self.rescale_factor.device != device:
            self.rescale_factor = self.rescale_factor.to(device)
        if self.tile_weights.device != device:
            self.tile_weights = self.tile_weights.to(device)

    def _denoise_local_tiles(self, x: Tensor, t_in: Tensor, c_in: CondDict, sd_model, N: int):
        """Tile shard: scatter and denoise this rank's tiles `[shard.begin, shard.end)`.  An interrupted rank stops its
        denoiser calls but keeps placeholder outputs (its inputs) so that the exchange still happens.
        Returns (outputs per local batch, interrupted)."""
        sh, g = self._shard, self._grid
        outs = []
        interrupted = False
        if sh.num_local > 0:
            self._tiles = engine.scatter_tiles(g, x, out=self._tiles, tile_begin=sh.begin, tile_end=sh.end, flags=self._blend_flags)
            icond_tiles, n_icond = None, 0
            if isinstance(c_in, dict):
                icond_full = self.get_icond(c_in)
                if tuple(icond_full.shape[2:]) == (self.h, self.w):
                    icond_tiles = engine.scatter_tiles(g, icond_full, tile_begin=sh.begin, tile_end=sh.end, flags=self._blend_flags)
                    n_icond = icond_full.shape[0]
            off = 0
            for batch_id, bboxes in enumerate(self.local_batched_bboxes):
                n_rep = len(bboxes)
                x_tile = self._tiles[off * N:(off + n_rep) * N]
                icond_tile = icond_tiles[off * n_icond:(off + n_rep) * n_icond] if icond_tiles is not None else None
                off += n_rep
                if interrupted or host.interrupted():
                    interrupted = True
                    outs.append(x_tile)
                    continue
                outs.append(self._denoise_tile_batch(sd_model, x_tile, n_rep, t_in, c_in, icond_tile, batch_id, N))
                self.update_pbar()
        return outs, interrupted

    def _grid_pass_sharded(self, x: Tensor, t_in: Tensor, c_in: CondDict, sd_model, N: int, C: int):
        """Tile shard (init_tile_shard): this rank denoises its contiguous chunk of the tile list, the eps tiles are
        all-gathered, and every rank runs the same ordered gaussian blend over all tiles -- bit-identical to the
        single-GPU result on every rank.  An interrupted rank stops its denoiser calls but still joins the all-gather
        (placeholder tiles) so that the collectives stay in lock-step, then returns None."""
        from .. import parallel
        sh, g = self._shard, self._grid
        outs, interrupted = self._denoise_local_tiles(x, t_in, c_in, sd_model, N)
        dt = outs[0].dtype if outs else x.dtype
        local = torch.zeros((sh.chunk * N, C, g.tile_h, g.tile_w), dtype=dt, device=x.device)
        if outs:
            torch.cat(outs, dim=0, out=local[:sh.num_local * N])
        gathered = parallel.gather_tile_outputs(local, self._shard_group)
        chunks = []
        for b in range(sh.num_chunks):
            nt = min(sh.chunk, sh.num_tiles - b * sh.chunk)
            chunks.append(gathered[b * sh.chunk * N:(b * sh.chunk + nt) * N])
        x_out = engine.blend_mixture(g, chunks, N, C, sh.chunk, self.tile_weights, self.rescale_factor, self.x_buffer,
                                     flags=self._blend_flags)
        return None if interrupted else x_out

    # ------------------------------------------------------------------ row-strip shard
    def init_tile_shard(self, group=None, fused: bool = True, mode: Optional[str] = None):
        """AbstractDiffusion.init_tile_shard; the default stays "replicate".  mode="strip": rank r denoises a run of tile rows
        and blends only its own canvas rows (row-window gaussian blend), exchanging only the overlapping tile rows and the
        latent halo -- bit-identical to one GPU.  Not with tiled noise inversion."""
        if mode == "strip" and self.noise_inverse_enabled:
            raise NotImplementedError(_STRIP_NO_INVERSION)
        return super().init_tile_shard(group, fused, mode)

    def _apply_strip(self, x_in: Tensor, x: Tensor, t_in: Tensor, c_in: CondDict, sd_model, N: int, C: int, custom_func):
        """One UNet call under the row-strip shard: this rank's tiles (`x` is valid on its strip plus latent halo), its custom
        regions, then the strip tail (`_strip_step`).  An interrupted rank still publishes, blends and signals (placeholder
        tiles), so the flag counters stay in lock-step, and then returns x_in."""
        outs, interrupted = [], False
        if self.enable_grid_bbox:
            self._blend_inputs_to(x.device)
            outs, interrupted = self._denoise_local_tiles(x, t_in, c_in, sd_model, N)
        done = None
        if custom_func is not None:
            # the region exchange (NCCL) comes before the tile exchange: its in-kernel waits then never sit in front of a collective
            done, interrupted = self._region_pass_sharded(x, custom_func, False, interrupted)
        out = self._strip_step(outs, x, N, C, done)
        return x_in if interrupted else out

    def _strip_latent_dtype(self, x_dtype: torch.dtype) -> torch.dtype:
        # the reference's feather overlay promotes to fp32 (fp32 mask, mixtureofdiffusers.py:124-128)
        fg = self.enable_custom_bbox and any(b.blend_mode == BlendMode.FOREGROUND for b in self.custom_bboxes)
        return torch.float32 if fg else x_dtype

    def _strip_blend(self, ex, x: Tensor, x_buffer: Optional[Tensor]):
        ex.blend_mixture(self._grid, self.tile_weights, self.rescale_factor, flags=self._blend_flags, x_buffer=x_buffer)

    def _region_composite_terms(self):
        return None, lambda bbox_id: self.custom_weights[bbox_id]

    def custom_apply_model(self, x_in: Tensor, t_in: Tensor, c_in: CondDict, bbox_id: int, bbox: CustomBBox) -> Tensor:
        """mixtureofdiffusers.py:181-196: a region goes through the un-hijacked `apply_model` with its own prompts."""
        sd_model = self._sd_model()
        if self.is_kdiff:
            return self.kdiff_custom_forward(x_in, t_in, c_in, bbox_id, bbox, forward_func=sd_model.apply_model_original_md)

        def forward_func(x, c, ts, unconditional_conditioning, *args, **kwargs) -> Tensor:
            # DDIM evaluates [uncond, cond] as one batch (p_sample_ddim)
            merged: CondDict = {}
            for k in c:
                if isinstance(c[k], list):
                    merged[k] = [torch.cat([unconditional_conditioning[k][i], c[k][i]]) for i in range(len(c[k]))]
                else:
                    merged[k] = torch.cat([unconditional_conditioning[k], c[k]])
            self.set_custom_controlnet_tensors(bbox_id, x.shape[0])
            self.set_custom_stablesr_tensors(bbox_id)
            return sd_model.apply_model_original_md(x, ts, merged)
        return self.ddim_custom_forward(x_in, c_in, bbox, ts=t_in, forward_func=forward_func)

    @torch.no_grad()
    def get_noise(self, x_in: Tensor, sigma_in: Tensor, cond_in: CondDict, step: int) -> Tensor:
        # the inverted latent is the full plan's: there is no host mask here, and an active tile reads kept pixels too
        self._full_plan_pass = True
        try:
            return self.apply_model_hijack(x_in, sigma_in, cond=cond_in, noise_inverse_step=step)
        finally:
            self._full_plan_pass = False
