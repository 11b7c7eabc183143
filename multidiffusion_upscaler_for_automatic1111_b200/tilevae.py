"""Tiled VAE with the reference's surface (scripts/tilevae.py: `VAEHook`, `GroupNormParam`,
`get_var_mean`, `custom_group_norm`, `crop_valid_region`, `build_task_queue`), H100-native
underneath.

What is different from the reference by design (80 GB of HBM, hand-written sm_90a kernels):
  * tiles, residuals and parked activations stay in HBM while they fit -- the reference stages every tile
    through host RAM (`.cpu()` at tilevae.py:534,610,641) and re-uploads it each round; when the tiles held at a
    slow-mode GroupNorm barrier exceed the budget (`VAEHook.max_resident_bytes`, default: the free device memory),
    the ones needed last wait in pinned host memory, copied on dedicated streams (`_Parking`);
  * GroupNorm statistics: one streaming read (`td_gn_stats`, fp32 Chan/Welford merge with
    warp shuffles) instead of `var_mean` on a reshaped copy;
  * GroupNorm apply + affine + SiLU: ONE fused pass (`td_gn_apply`) instead of
    batch_norm, `*= weight`, `+= bias`, `silu_` (4 read+write passes, tilevae.py:237-244,:104);
  * tile crop and valid-region paste are `td_copy_region` launches; the result canvas is
    allocated once in the network dtype (the reference's fp32 canvas + final cast is a
    lossless round trip for fp16/bf16 tile outputs);
  * no per-tile NaN test (each one is a full read + host sync, tilevae.py:625): the result
    is checked once at the end and the estimator keeps its NaN fallback.
  * fp16 / bf16 networks run channels-last with every convolution and the attention GEMMs on the tensor cores
    (wgmma, csrc/td_conv.cu) through `vae_engine.TensorCoreBackend`; fp32 networks keep the host application's
    modules for the dense ops (`vae_engine.ModuleBackend`).
The network is compiled once into an op program (`vae_engine.compile_program`); GroupNorm sites are barriers between
tiles unless fast mode froze their statistics.
"""
from __future__ import annotations

import ctypes
import math
import time
import weakref
from typing import Callable, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import engine, host
from ._cabi import check, current_stream_ptr, dtype_code, lib

NUM_GROUPS = 32
GN_EPS = 1e-6


# --------------------------------------------------------------------------- kernels (tensor wrappers)
def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor: the tiled-VAE path has no CPU fallback (got {t.device})")


def _segment_stats(x: torch.Tensor, nseg: int, seg_len: int, unbiased: bool, want_minmax: bool = False):
    _require_cuda(x, "activation")
    dev = x.device
    ws_bytes = lib.td_gn_stats_workspace_bytes(nseg, seg_len, dtype_code(x.dtype))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    mean = torch.empty(nseg, dtype=torch.float32, device=dev)
    var = torch.empty(nseg, dtype=torch.float32, device=dev)
    lo = torch.empty(nseg, dtype=torch.float32, device=dev) if want_minmax else None
    hi = torch.empty(nseg, dtype=torch.float32, device=dev) if want_minmax else None
    with torch.cuda.device(dev):
        check(lib.td_gn_stats(x.data_ptr(), nseg, seg_len, dtype_code(x.dtype), int(unbiased), ws.data_ptr(), ws_bytes,
                              mean.data_ptr(), var.data_ptr(), lo.data_ptr() if want_minmax else None,
                              hi.data_ptr() if want_minmax else None, current_stream_ptr(dev)))
    return (var, mean, lo, hi) if want_minmax else (var, mean)


def get_var_mean(input: torch.Tensor, num_groups: int, eps: float = 1e-6):
    """tilevae.py:207-215: biased variance and mean per (batch, group), fp32 [b*num_groups] each."""
    b, c = input.size(0), input.size(1)
    cpg = int(c / num_groups)
    x = input.contiguous()
    seg_len = cpg * int(np.prod(x.shape[2:]))
    return _segment_stats(x, int(b * num_groups), seg_len, unbiased=False)


def _affine32(layer_weight, layer_bias, device):
    g = layer_weight.detach().to(device=device, dtype=torch.float32).contiguous() if layer_weight is not None else None
    b = layer_bias.detach().to(device=device, dtype=torch.float32).contiguous() if layer_bias is not None else None
    return g, b


def custom_group_norm(input: torch.Tensor, num_groups: int, mean: torch.Tensor, var: torch.Tensor, weight=None, bias=None,
                      eps: float = 1e-6, act: bool = False, inplace: bool = False) -> torch.Tensor:
    """tilevae.py:218-245 (+ optional fused SiLU): group norm with externally supplied statistics.

    mean / var: [num_groups] (shared by the batch, as the reference's merged statistics are)
    or [b*num_groups]."""
    _require_cuda(input, "activation")
    b, c = input.size(0), input.size(1)
    x = input.contiguous()
    hw = int(np.prod(x.shape[2:]))
    per_batch = mean.numel() == b * num_groups and b > 1
    if mean.numel() not in (num_groups, b * num_groups):
        raise ValueError(f"statistics have {mean.numel()} entries; expected {num_groups} or {b * num_groups}")
    mean32 = mean.to(device=x.device, dtype=torch.float32).contiguous()
    var32 = var.to(device=x.device, dtype=torch.float32).contiguous()
    gamma, beta = weight, bias
    if gamma is not None and gamma.dtype != torch.float32:
        gamma, beta = _affine32(gamma, beta, x.device)
    out = x if inplace else torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.td_gn_apply(x.data_ptr(), out.data_ptr(), b, c, hw, dtype_code(x.dtype), num_groups, mean32.data_ptr(),
                              var32.data_ptr(), int(per_batch), gamma.data_ptr() if gamma is not None else None,
                              beta.data_ptr() if beta is not None else None, float(eps), int(act), current_stream_ptr(x.device)))
    return out


def copy_region(src: torch.Tensor, dst: torch.Tensor) -> None:
    """dst[...] = src[...] for two 4-D views [N, C, rows, cols] whose last dim has stride 1 and whose
    (N, C) dims collapse to one plane stride (contiguous parents).  One td_copy_region launch."""
    _require_cuda(src, "src"); _require_cuda(dst, "dst")
    assert src.shape == dst.shape and src.dtype == dst.dtype and src.dim() == 4
    n, c, rows, cols = src.shape
    for t in (src, dst):
        assert t.stride(3) == 1 and (n == 1 or t.stride(0) == c * t.stride(1)), "unsupported view layout"
    with torch.cuda.device(dst.device):
        check(lib.td_copy_region(src.data_ptr(), dst.data_ptr(), n * c, rows, cols, src.stride(1), src.stride(2), dst.stride(1),
                                 dst.stride(2), dtype_code(src.dtype), current_stream_ptr(dst.device)))


def crop_valid_region(x: torch.Tensor, input_bbox, target_bbox, is_decoder: bool) -> torch.Tensor:
    """tilevae.py:248-259 (a view; the paste that follows is the copy)."""
    padded = [i * 8 if is_decoder else i // 8 for i in input_bbox]
    margin = [target_bbox[i] - padded[i] for i in range(4)]
    return x[:, :, margin[2]:x.size(2) + margin[3], margin[0]:x.size(3) + margin[1]]


def nearest_exact_indices(in_size: int, scale_factor: float):
    """Output size and source indices of F.interpolate(mode='nearest-exact', scale_factor=s):
    out = floor(in * s); src = min(floor((dst + 0.5) * float32(1 / s)), in - 1) (ATen UpSample)."""
    out = int(math.floor(float(in_size) * scale_factor))
    inv = np.float32(1.0 / scale_factor)
    idx = np.floor((np.arange(out, dtype=np.float32) + np.float32(0.5)) * inv).astype(np.int64)
    return out, np.minimum(idx, in_size - 1).astype(np.int32)


def fast_mode_estimator_input(z: torch.Tensor, tile_size: int) -> torch.Tensor:
    """tilevae.py:545-559 on the device: nearest-exact resample, per-channel re-standardisation
    (unbiased std) and clamp to z's range; z is read once for its statistics."""
    _require_cuda(z, "z")
    z = z.contiguous()
    B, C, H, W = z.shape
    scale = tile_size / max(H, W)
    oh, sy = nearest_exact_indices(H, scale)
    ow, sx = nearest_exact_indices(W, scale)
    dev = z.device
    sy_d, sx_d = torch.from_numpy(sy).to(dev), torch.from_numpy(sx).to(dev)
    ds = torch.empty((B, C, oh, ow), dtype=z.dtype, device=dev)
    with torch.cuda.device(dev):
        check(lib.td_resample_nearest(z.data_ptr(), ds.data_ptr(), B * C, H, W, oh, ow, sy_d.data_ptr(), sx_d.data_ptr(),
                                      dtype_code(z.dtype), current_stream_ptr(dev)))

    def channel_stats(t, hw, want_minmax):
        out = _segment_stats(t, B * C, hw, unbiased=True, want_minmax=want_minmax)
        var, mean = out[0].view(B, C), out[1].view(B, C)
        if B > 1:   # torch.std_mean over dims [0, 2, 3]: merge the per-(b, c) moments (equal counts)
            # shifted by the first image's mean: equal means merge to exactly that mean (a plain fp32 mean of three
            # equal values can miss it by an ulp, and a channel that is constant over the batch would get std > 0)
            m = mean[0] + (mean - mean[0]).mean(dim=0)
            m2 = (var * (hw - 1)).sum(dim=0) + hw * ((mean - m) ** 2).sum(dim=0)
            var, mean = m2 / (B * hw - 1), m
        else:
            var, mean = var[0], mean[0]
        return (var.sqrt(), mean) + ((out[2].min().view(1), out[3].max().view(1)) if want_minmax else ())

    std_old, mean_old, lo, hi = channel_stats(z, H * W, True)
    std_new, mean_new = channel_stats(ds, oh * ow, False)
    # the reference's statistics are tensors of z.dtype: round them the same way
    rt = lambda t: t.to(z.dtype).float().contiguous()
    mean_new, std_new, mean_old, std_old = rt(mean_new), rt(std_new), rt(mean_old), rt(std_old)
    with torch.cuda.device(dev):
        check(lib.td_affine_clamp(ds.data_ptr(), B, C, oh * ow, dtype_code(ds.dtype), mean_new.data_ptr(), std_new.data_ptr(),
                                  mean_old.data_ptr(), std_old.data_ptr(), lo.data_ptr(), hi.data_ptr(), current_stream_ptr(dev)))
    return ds


# --------------------------------------------------------------------------- program views / statistics merge
def build_task_queue(net, is_decoder):
    """The compiled program in the reference's task-queue vocabulary (tilevae.py:107-204 names): a read-only VIEW for
    callers that inspect the queue (logging, tests); execution uses `vae_engine.Program` directly."""
    from . import vae_engine as ve
    prog = ve.compile_program(net, is_decoder)
    queue, first = [], True
    for op in prog.ops:
        if isinstance(op, ve.Skip):
            queue.append(('store_res', op.module if op.module is not None else (lambda x: x)))
        elif isinstance(op, ve.Norm):
            queue.append(('pre_norm', op.module))
            if op.act:
                queue.append(('silu', lambda x: F.silu(x, inplace=True)))
        elif isinstance(op, ve.Conv):
            if first:
                name = 'conv_in'
            elif op.upsample_first:
                name = 'upsample'
            elif op.downsample:
                name = 'downsample'
            elif op.module is getattr(net, 'conv_out', None):
                name = 'conv_out'
            else:
                name = 'conv2' if op.add_skip else 'conv1'
            queue.append((name, op.module))
            if op.add_skip:
                queue.append(['add_res', None])
        elif isinstance(op, ve.Attention):
            queue.append(('attn', op.module))
            queue.append(['add_res', None])
        elif isinstance(op, ve.Tanh):
            queue.append(('tanh', torch.tanh))
        first = False
    return queue


class GroupNormParam:
    """One GroupNorm round (tilevae.py:289-361): per-tile statistics in, merged statistics out.

    Merge rule of the reference (:320-335): weights p_i = pixels_i / sum(pixels); var = sum p_i var_i,
    mean = sum p_i mean_i (no between-tile term).  With a process group (tile shard over ranks) the weighted sums
    are all-reduced, so every rank applies the statistics of ALL tiles; every rank takes part in every round, tiles
    or not -- the number of rounds follows from the program, no host agreement is needed."""

    def __init__(self, group=None, sharded: bool = False):
        self.group, self.sharded = group, sharded
        self.var_list, self.mean_list, self.pixel_list = [], [], []

    def add(self, var: torch.Tensor, mean: torch.Tensor, pixels: int):
        self.var_list.append(var)
        self.mean_list.append(mean)
        self.pixel_list.append(pixels)

    def add_tile(self, tile, layer=None):
        """Reference-style entry point: statistics of an NCHW tile (fp32: no fp16 overflow branch needed, :300-304)."""
        var, mean = get_var_mean(tile, NUM_GROUPS)
        self.add(var, mean, tile.shape[2] * tile.shape[3])

    def summary(self, stat_len: Optional[int] = None, device=None, images: int = 1):
        """-> (mean, var) fp32 tensors, or None when no tile contributed anywhere.

        images > 1: each tile's statistics hold `images` images one after the other (a batched tensor-core pass) and
        every image is merged on its own, with the operations and the all-reduce its one-image pass would run, so
        its statistics are the same bits.  stat_len then counts all images."""
        if images == 1:
            return self._merge(self.var_list, self.mean_list, stat_len, device)
        per = [self._merge([v.view(images, -1)[j] for v in self.var_list], [m.view(images, -1)[j] for m in self.mean_list],
                           None if stat_len is None else int(stat_len) // images, device) for j in range(images)]
        if any(p is None for p in per):
            return None
        return torch.cat([p[0] for p in per]), torch.cat([p[1] for p in per])

    def _merge(self, var_list, mean_list, stat_len, device):
        if not self.sharded:
            if not var_list:
                return None
            var, mean = torch.vstack(var_list), torch.vstack(mean_list)
            px = torch.tensor(self.pixel_list, dtype=torch.float32, device=var.device)
            px = (px / px.sum()).unsqueeze(1)
            return torch.sum(mean * px, dim=0), torch.sum(var * px, dim=0)
        import torch.distributed as dist
        if var_list:
            px = torch.tensor(self.pixel_list, dtype=torch.float32, device=var_list[0].device).unsqueeze(1)
            packed = torch.cat([(torch.vstack(var_list) * px).sum(0), (torch.vstack(mean_list) * px).sum(0), px.sum().view(1)])
        else:
            packed = torch.zeros(2 * int(stat_len) + 1, dtype=torch.float32, device=device)
        dist.all_reduce(packed, group=self.group)
        k = (packed.numel() - 1) // 2
        return packed[k:2 * k] / packed[-1], packed[:k] / packed[-1]


# --------------------------------------------------------------------------- parking
def _dense_bytes(t: torch.Tensor) -> torch.Tensor:
    """A uint8 view of the memory of a dense tensor in any dimension order (the module backend's convolutions may
    return channels-last tensors): a parked tensor comes back with its own strides, so later ops see the same layout."""
    p = t.permute(sorted(range(t.dim()), key=lambda d: -t.stride(d)))
    assert p.is_contiguous(), f"cannot park a tensor with strides {t.stride()}"
    return p.reshape(-1).view(torch.uint8)


class _Parking:
    """Pinned host homes for the tiles a residency plan parks, and the two copy streams that move them (the H100 has a
    copy engine per direction).  Copies overlap with the kernels of the tiles being computed.

      * park: after the tile's statistics kernel, its `act` / `skip` go to its pinned buffer on the device-to-host
        stream; the device blocks are handed back with record_stream, so the caching allocator reuses them only once
        the copy has read them.  A shortcut whose host copy is still current (the block input of an identity shortcut,
        parked at norm1, is the shortcut at norm2) is not copied again.  Buffer layout: shortcut at 0, activation after
        it; an aliased pair is one region.
      * resume: the tile's upload (issued before, while the previous tile computed) is waited on by the compute stream,
        the deferred barrier norm is applied, and the upload of the next parked tile in the visiting order is issued.
    Buffers are pageable host memory registered with cudaHostRegister (exact sizes), released by `close`."""

    def __init__(self, device, sizes, stats: dict):
        self.device, self.sizes, self.stats = device, sizes, stats
        self.d2h = torch.cuda.Stream(device)
        self.h2d = torch.cuda.Stream(device)
        self.buf = {}          # tile -> registered uint8 host tensor
        self.slot = {}         # tile -> {"act": (offset, shape, strides, dtype), "skip": ..., "written": Event}
        self.home = set()      # tiles whose state is on the host
        self.uploads = {}      # tile -> (act, skip, Event): device tensors being filled on the upload stream
        self.pending = {}      # tile -> (norm op, mean, var) to apply on resume
        self.current = {}      # tile -> weakref of the device shortcut whose host copy is current
        self.last_written = None

    def parked(self, i) -> bool:
        return i in self.home

    def _buffer(self, i):
        if i not in self.buf:
            t0 = time.perf_counter()
            t = torch.empty(self.sizes[i], dtype=torch.uint8)
            err = int(torch.cuda.cudart().cudaHostRegister(t.data_ptr(), t.numel(), 0))
            if err != 0:
                raise RuntimeError(f"[Tiled VAE]: pinning {t.numel()} bytes of host memory failed (cudaError {err})")
            self.buf[i] = t
            self.stats["host_bytes"] += t.numel()
            self.stats["pin_s"] += time.perf_counter() - t0
        return self.buf[i]

    def park(self, i, st, site: int) -> None:
        buf = self._buffer(i)
        if self.last_written is not None:
            # one write-back in flight: the caching allocator frees a parked block on the host's side once its copy is
            # done, so without this wait a run ahead of the copy engine would keep every parked tile allocated
            self.last_written.synchronize()
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))
        self.d2h.wait_event(ready)
        ref = self.current.pop(i, None)
        slot, copied, off = {}, [], 0
        with torch.cuda.stream(self.d2h):
            if st.skip is not None:
                if ref is None or ref() is not st.skip:
                    copied.append((0, st.skip))
                slot["skip"] = (0, st.skip.shape, st.skip.stride(), st.skip.dtype)
                off = st.skip.numel() * st.skip.element_size()
            if st.skip is not None and st.act is st.skip:
                slot["act"] = slot["skip"]
            else:
                copied.append((off, st.act))
                slot["act"] = (off, st.act.shape, st.act.stride(), st.act.dtype)
            for o, t in copied:
                n = t.numel() * t.element_size()
                buf[o:o + n].copy_(_dense_bytes(t), non_blocking=True)
                t.record_stream(self.d2h)
                self.stats["d2h_bytes"] += n
            slot["written"] = torch.cuda.Event()
            slot["written"].record(self.d2h)
        self.slot[i] = slot
        self.last_written = slot["written"]
        st.act = st.skip = None
        self.home.add(i)
        per_site = self.stats["tiles_parked"]
        per_site[site] = per_site.get(site, 0) + 1

    def defer(self, i, norm, mean, var) -> None:
        self.pending[i] = (norm, mean, var)

    def _upload(self, i) -> None:
        if i in self.uploads or i not in self.home:
            return
        slot, buf = self.slot[i], self.buf[i]
        alloc = lambda d: torch.empty_strided(d[1], d[2], dtype=d[3], device=self.device)     # the parked tensor's strides
        skip = alloc(slot["skip"]) if "skip" in slot else None
        aliased = "skip" in slot and slot["act"] is slot["skip"]
        act = skip if aliased else alloc(slot["act"])
        # the blocks come from the compute stream's pool: kernels queued before may still read their previous tenant
        free = torch.cuda.Event()
        free.record(torch.cuda.current_stream(self.device))
        self.h2d.wait_event(free)
        self.h2d.wait_event(slot["written"])
        with torch.cuda.stream(self.h2d):
            for t, desc in ((skip, slot.get("skip")), (None if aliased else act, slot["act"])):
                if t is None:
                    continue
                n = t.numel() * t.element_size()
                _dense_bytes(t).copy_(buf[desc[0]:desc[0] + n], non_blocking=True)
                self.stats["h2d_bytes"] += n
            done = torch.cuda.Event()
            done.record(self.h2d)
        self.uploads[i] = (act, skip, done)

    def resume(self, ex, i, st, ahead) -> None:
        """Before tile i computes: its state back on the device, and the next parked tile of `ahead` on its way."""
        self._upload(i)
        nxt = next((j for j in ahead if j in self.home), None)
        if nxt is not None:
            self._upload(nxt)
        if i not in self.home:
            return
        act, skip, done = self.uploads.pop(i)
        torch.cuda.current_stream(self.device).wait_event(done)
        self.home.discard(i)
        st.act, st.skip = act, skip
        if skip is not None:
            self.current[i] = weakref.ref(skip)
        if i in self.pending:
            ex.apply_barrier(st, *self.pending.pop(i))

    def close(self) -> None:
        """Drain both copy streams (also after an interrupt), then release the pinned buffers."""
        self.d2h.synchronize()
        self.h2d.synchronize()
        self.uploads.clear()
        self.pending.clear()
        for t in self.buf.values():
            torch.cuda.cudart().cudaHostUnregister(t.data_ptr())
        self.buf.clear()


# --------------------------------------------------------------------------- the hook
def pick_images_per_pass(n: int, fits: Callable[[int], bool]) -> int:
    """The largest k <= n with fits(k) (k > 1 only: one image at a time is the schedule that always runs), else 1."""
    for k in range(n, 1, -1):
        if fits(k):
            return k
    return 1


def shard_tiles(tiles, world: int, rank: int) -> List[int]:
    """The tiles rank `rank` of a `world`-rank tile shard runs out of the tiles a pass runs (in order): every world-th, so
    the ranks stay balanced when an inpaint mask skips tiles."""
    return list(tiles)[rank::world]


class VAEHook:

    def __init__(self, net, tile_size, is_decoder: bool, fast_decoder: bool, fast_encoder: bool, color_fix: bool, to_gpu: bool = False):
        self.net = net
        self.tile_size = tile_size
        self.is_decoder = is_decoder
        self.fast_mode = (fast_encoder and not is_decoder) or (fast_decoder and is_decoder)
        self.color_fix = color_fix and not is_decoder
        self.to_gpu = to_gpu
        self.pad = 11 if is_decoder else 32
        self.verbose = False
        self.backend_name = None      # which backend ran the last call ("wgmma" / "modules")
        # Slow-mode tiles kept in GPU memory at a GroupNorm barrier may hold at most this many bytes; the others wait in
        # pinned host memory.  None: the free device memory at the start of the call, less the working reserve.
        self.max_resident_bytes: Optional[int] = None
        self.last_park_stats: Optional[dict] = None    # what the last call parked (see _run_tiles)
        # Tensor-core backend: images of a batch that go through the tiles together, each with its own GroupNorm statistics,
        # fast-mode estimate and color fix (bit-identical to one image at a time).  None: the largest count whose working set
        # fits in GPU memory and whose tiles all stay resident under the parking budget (`_images_per_pass`); 1: one pass per
        # image.  The count used is last_park_stats["images_per_pass"].
        self.images_per_pass: Optional[int] = None
        # Seamless tiling: the latent / image is periodic along x (y).  The tiles are then cut around the circle and read
        # their halo from the opposite edge, so a wrapped decode of a seamless latent has no seam (td_vae_split_tiles' `wrap`).
        self.wrap_x: bool = False
        self.wrap_y: bool = False
        # Inpainting (fast-mode decoder): [P, 1, oh, ow] image-space mask, 1 = keep the original, and the [P, out_c, oh, ow]
        # canvas the skipped tiles keep (None: zeros).  Set with `set_inpaint_mask`.
        self.inpaint_mask: Optional[torch.Tensor] = None
        self.inpaint_fill: Optional[torch.Tensor] = None
        self._program = None
        self._shard_group = None
        self._shard_world = 1
        self._shard_rank = 0

    def init_tile_shard(self, group=None):
        """Shard the VAE tiles over the ranks of `group` (one process per GPU): rank r runs tiles i with
        i % world == r; GroupNorm statistics (slow mode) are all-reduced per round and the disjoint output
        regions are exchanged with one all-gather.  New: the reference is single-device."""
        import torch.distributed as dist
        self._shard_group = group
        self._shard_world = dist.get_world_size(group)
        self._shard_rank = dist.get_rank(group)

    def set_inpaint_mask(self, mask: Optional[torch.Tensor], fill: Optional[torch.Tensor] = None) -> None:
        """Decode only the tiles an inpaint mask reaches, in every later call until `set_inpaint_mask(None)`.  New: the
        reference decodes every tile.

        mask: image-space, 1 = keep the original (the host's blurred overlay mask, inverted and scaled to [0, 1]), [oh, ow],
        [1, oh, ow] or [N, 1, oh, ow], fp16 / bf16 / fp32 on the device.  A tile runs when one mask element in its output
        rectangle is not exactly 1.0 (NaN included); with per-image masks, when one image of its pass reaches it.
        fill: None (zeros) or [N or 1, out_c, oh, ow] in the network's dtype on its device, e.g. the init image in [-1, 1]:
        what the skipped rectangles of the result hold.  An active tile's rectangle is bit-identical to an unmasked call.

        Fast-mode decoders only: every GroupNorm site is then frozen before the tiles run, so skipping a tile changes no
        other tile.  An image whose estimate met a NaN (slow mode) runs all its tiles.  Refused before any change:
        NotImplementedError for an encoder or slow mode, ValueError for a bad shape or dtype."""
        if mask is None:
            self.inpaint_mask = self.inpaint_fill = None
            return
        if not self.is_decoder:
            raise NotImplementedError("[Tiled VAE]: inpainting skips decoder tiles only; the encoder needs the whole latent")
        if not self.fast_mode:
            raise NotImplementedError("[Tiled VAE]: inpainting needs the fast decoder: slow mode's GroupNorm barriers need every tile")
        floats = (torch.float16, torch.bfloat16, torch.float32)
        if not isinstance(mask, torch.Tensor) or mask.dtype not in floats:
            raise ValueError(f"inpaint mask must be an fp16 / bf16 / fp32 tensor, got {getattr(mask, 'dtype', type(mask))}")
        shape = tuple(mask.shape)
        ok = (len(shape) == 2 or (len(shape) == 3 and shape[0] == 1) or (len(shape) == 4 and shape[1] == 1 and shape[0] >= 1))
        if not ok or mask.numel() == 0:
            raise ValueError(f"inpaint mask shape {shape}: expected [oh, ow], [1, oh, ow] or [N, 1, oh, ow]")
        if fill is not None:
            if not isinstance(fill, torch.Tensor) or fill.dtype not in floats:
                raise ValueError(f"inpaint fill must be an fp16 / bf16 / fp32 tensor, got {getattr(fill, 'dtype', type(fill))}")
            if fill.dim() != 4 or fill.numel() == 0 or tuple(fill.shape[-2:]) != shape[-2:]:
                raise ValueError(f"inpaint fill shape {tuple(fill.shape)}: expected [N or 1, out_c, {shape[-2]}, {shape[-1]}]")
        for what, t in (("mask", mask), ("fill", fill)):
            if t is not None and not t.is_cuda:
                raise ValueError(f"inpaint {what} must be on the device, got {t.device}")
        self.inpaint_mask = mask.reshape(-1, 1, shape[-2], shape[-1]).contiguous()
        self.inpaint_fill = fill.contiguous() if fill is not None else None

    def _inpaint_inputs(self, N, out_c, oh, ow, device, dtype):
        """(mask, fill) checked against this call, before any tile runs."""
        mask, fill = self.inpaint_mask, self.inpaint_fill
        if mask.shape[0] not in (1, N) or tuple(mask.shape[-2:]) != (oh, ow) or mask.device != device:
            raise ValueError(f"inpaint mask {tuple(mask.shape)} on {mask.device} does not match this call: {N} images of {oh} x {ow} "
                             f"on {device}")
        if fill is not None and (fill.shape[0] not in (1, N) or tuple(fill.shape[1:]) != (out_c, oh, ow) or fill.dtype != dtype
                                 or fill.device != device):
            raise ValueError(f"inpaint fill {tuple(fill.shape)} {fill.dtype} on {fill.device} does not match this call: "
                             f"[{N} or 1, {out_c}, {oh}, {ow}] {dtype} on {device}")
        return mask, fill

    def __call__(self, x):
        original_device = next(self.net.parameters()).device
        try:
            if self.to_gpu:
                self.net = self.net.to(host.device())
            B, C, H, W = x.shape
            if max(H, W) <= self.pad * 2 + self.tile_size and not self._wrap():   # a wrapped seam always gets its halo
                if self.verbose:
                    print("[Tiled VAE]: the input size is tiny and unnecessary to tile.")
                return self.net.original_forward(x)
            return self.vae_tile_forward(x)
        finally:
            self.net = self.net.to(original_device)

    def get_best_tile_size(self, lowerbound, upperbound):
        return lib.td_vae_best_tile_size(int(lowerbound), int(upperbound))

    def _wrap(self) -> int:
        return (1 if self.wrap_x else 0) | (2 if self.wrap_y else 0)

    def split_tiles(self, h, w):
        """tilevae.py:405-462 -> (tile_input_bboxes, tile_output_bboxes), each [x1, x2, y1, y2].  On a wrapped axis the
        input bboxes are in unwrapped coordinates."""
        args = (int(h), int(w), int(self.tile_size), int(self.pad), int(self.is_decoder), self._wrap())
        n = check(lib.td_vae_split_tiles(*args, None, None, 0))
        ib = np.empty((n, 4), dtype=np.int32)
        ob = np.empty((n, 4), dtype=np.int32)
        p = ctypes.POINTER(ctypes.c_int32)
        check(lib.td_vae_split_tiles(*args, ib.ctypes.data_as(p), ob.ctypes.data_as(p), n))
        return ib.tolist(), ob.tolist()

    def _cheap_fallback(self, z, device, dtype):
        """What the reference returns when interrupted before any tile finished (tilevae.py:573-577, :656): the cheap
        latent -> RGB approximation, nearest-exact x8.  Only a decoder has one; the encoder raises like the reference
        (None.to(...))."""
        approx = host.get_cheap_approximation()
        if approx is None or not self.is_decoder:
            raise RuntimeError("[Tiled VAE]: interrupted before any tile finished and no cheap approximation is available")
        with torch.no_grad():
            out = torch.cat([F.interpolate(approx(x).unsqueeze(0), scale_factor=8, mode="nearest-exact") for x in z], dim=0)
        return out.to(device=device, dtype=dtype)

    @torch.no_grad()
    def vae_tile_forward(self, z):
        """tilevae.py:509-656, device-resident, on the compiled program."""
        from . import vae_engine as ve
        param = next(self.net.parameters())
        device, dtype = param.device, param.dtype
        if device.type != "cuda":
            raise RuntimeError(f"VAEHook: network is on {device}; the H100 tiled-VAE path has no CPU fallback")
        net, tile_size, is_decoder = self.net, self.tile_size, self.is_decoder
        z = z.detach().to(device=device, dtype=dtype).contiguous()
        N, height, width = z.shape[0], z.shape[2], z.shape[3]
        net.last_z_shape = z.shape
        in_bboxes, out_bboxes = self.split_tiles(height, width)
        if self._program is None or self._program.cache.get("net_id") != id(net):
            self._program = ve.compile_program(net, is_decoder)
            self._program.cache["net_id"] = id(net)
        program = self._program
        backend = ve.pick_backend(program, device, dtype)
        self.backend_name = backend.name
        est_in = fast_mode_estimator_input(z, tile_size) if self.fast_mode else None

        sharded = self._shard_world > 1
        num_tiles = len(in_bboxes)
        mine = shard_tiles(range(num_tiles), self._shard_world, self._shard_rank)
        my_in = [in_bboxes[i] for i in mine]
        out_c = [op for op in program.ops if isinstance(op, ve.Conv)][-1].module.out_channels
        oh, ow = (height * 8, width * 8) if is_decoder else (height // 8, width // 8)
        mask, fill = self._inpaint_inputs(N, out_c, oh, ow, device, dtype) if self.inpaint_mask is not None else (None, None)
        if fill is None:
            result = torch.zeros((N, out_c, oh, ow), dtype=dtype, device=device)   # zeros: a partial (interrupted) result reads 0 elsewhere
        else:
            result = torch.empty((N, out_c, oh, ow), dtype=dtype, device=device)
            for n in range(N) if fill.shape[0] == 1 and N > 1 else (None,):
                copy_region(fill, result if n is None else result[n:n + 1])
        # budget / reserve: bytes (None when no barrier); host_bytes: pinned host memory (its peak: buffers live until the
        # call ends); d2h / h2d_bytes: bytes copied each way; pin_s: seconds spent pinning; tiles_parked: {site: tiles}
        # images_per_pass: images that went through the tiles together; tiles_run: tiles this rank ran, summed over the
        # passes; tiles_skipped: tiles no rank ran because the inpaint mask does not reach them, summed over the passes
        self.last_park_stats = {"budget": None, "reserve": None, "host_bytes": 0, "d2h_bytes": 0, "h2d_bytes": 0, "pin_s": 0.0,
                                "tiles_parked": {}, "tiles_run": 0, "tiles_skipped": 0}
        k = self._images_per_pass(program, backend, z, my_in) if isinstance(backend, ve.TensorCoreBackend) else N
        self.last_park_stats["images_per_pass"] = k
        # (images, tiles) whose output regions the shard exchanges: every tile of the batch, or per pass the tiles it ran
        exchanged = [] if mask is not None else [(slice(0, N), list(range(num_tiles)))]

        def one_pass(img):
            """Tiles finished by one pass over images `img`; None when the estimate of a batched pass met a NaN."""
            ex = ve.Executor(program, backend)
            if est_in is not None:
                if isinstance(backend, ve.TensorCoreBackend) and img.stop - img.start > 1:
                    if not ex.estimate(backend.load(est_in[img]), self.color_fix, report=False):
                        return None
                else:
                    ex.estimate(backend.load(est_in[img]), self.color_fix)
            tiles = list(range(num_tiles))
            if mask is not None:
                # frozen sites only: a tile's output then depends on its own input and the pass's images.  A pass with a
                # barrier (an estimate that met a NaN) needs every tile's statistics and runs them all
                if ex.barrier_sites() == 0:
                    tiles = np.flatnonzero(engine.vae_active_tiles(mask if mask.shape[0] == 1 else mask[img], out_bboxes)).tolist()
                exchanged.append((img, tiles))
            run = shard_tiles(tiles, self._shard_world, self._shard_rank)
            self.last_park_stats["tiles_run"] += len(run)
            self.last_park_stats["tiles_skipped"] += num_tiles - len(tiles)
            return self._run_tiles(ex, backend, z[img], result[img], [in_bboxes[i] for i in run], [out_bboxes[i] for i in run])

        finished = 0
        for start in range(0, N, k):
            done = one_pass(slice(start, min(start + k, N)))
            if done is None:
                # an image whose estimate met a NaN runs without frozen statistics while the others keep theirs: one pass
                # per image, as a one-image schedule runs them (the estimate is the same on every rank of a tile shard)
                for n in range(start, min(start + k, N)):
                    finished += one_pass(slice(n, n + 1))
                    if host.interrupted():
                        break
            else:
                finished += done
            if host.interrupted():
                break
        interrupted = host.interrupted()
        if sharded:
            self._exchange_regions(result, out_bboxes, exchanged)
        if finished == 0 and mine and interrupted:
            return self._cheap_fallback(z, device, dtype)
        if not interrupted and torch.isnan(result).any():
            raise RuntimeError("[Tiled VAE]: NaN in the result (the reference's test_for_nans, tilevae.py:625)")
        return result

    def _run_tiles(self, ex, backend, z, result, in_bboxes, out_bboxes) -> int:
        """All tiles of one image (or image batch) through the program: rounds separated by the barrier sites.  An input
        tile is loaded on its first visit.  When the tiles held at a barrier do not all fit in GPU memory, the ones the
        residency plan picks wait in pinned host memory until their next visit (`_Parking`); when they fit, nothing is
        copied."""
        from . import vae_engine as ve
        num_tiles = len(in_bboxes)
        states = [ve.TileState(None) for _ in range(num_tiles)]
        sharded = self._shard_world > 1
        rounds = ex.barrier_sites()
        barriers = [op for op in ex.program.ops if isinstance(op, ve.Norm) and ex.frozen[op.site] is None]
        plan = self._park_plan(ex, backend, z, in_bboxes, barriers)
        pk = _Parking(z.device, plan[1], self.last_park_stats) if plan is not None else None
        done = 0
        forward = True
        try:
            for rnd in range(rounds + 1):
                if host.interrupted():
                    break
                collect = GroupNormParam(self._shard_group, sharded)
                site = None
                order = list(range(num_tiles)) if forward else list(range(num_tiles - 1, -1, -1))   # the reference's zig-zag (:599)
                park_now = set(plan[0][rnd]) if pk is not None and rnd < rounds else ()
                for k, i in enumerate(order):
                    if host.interrupted():
                        break
                    st = states[i]
                    if st is None:
                        continue
                    if pk is not None:
                        pk.resume(ex, i, st, [j for j in order[k + 1:] if states[j] is not None])
                    if st.act is None:
                        b = in_bboxes[i]
                        st.act = backend.load_wrap(z, b) if self._wrap() else backend.load(z[:, :, b[2]:b[3], b[0]:b[1]])
                    stop = ex.run(st)
                    if stop is None:
                        backend.paste(st.act, result, in_bboxes[i], out_bboxes[i], self.is_decoder)
                        states[i] = None
                        done += 1
                    else:
                        site = stop
                        var, mean = backend.stats(st.act)
                        collect.add(var, mean, backend.pixels(st.act))
                        if i in park_now:
                            pk.park(i, st, stop.site)
                forward = not forward
                if rnd == rounds or host.interrupted():
                    break
                if site is None and sharded:      # a rank without tiles still joins the round's all-reduce
                    site = barriers[rnd]
                if site is None:
                    break
                stat_len = NUM_GROUPS * z.shape[0]
                merged = collect.summary(stat_len, z.device, z.shape[0] if isinstance(backend, ve.TensorCoreBackend) else 1)
                if merged is None:
                    break
                mean, var = merged
                for i, st in enumerate(states):
                    if st is None:
                        continue
                    if pk is not None and pk.parked(i):
                        pk.defer(i, site, mean, var)      # normalised when it is back on the device
                    else:
                        ex.apply_barrier(st, site, mean, var)
        finally:
            if pk is not None:
                pk.close()
        return done

    def _park_plan(self, ex, backend, z, in_bboxes, barriers):
        """None when every tile fits at every barrier; else (tiles parked at each barrier, pinned bytes per parked tile).

        Budget for the resident tiles: the free device memory (driver + the caching allocator's unused blocks) less
        the largest working set of one tile and two tiles' parked bytes (one upload and one write-back in flight);
        `max_resident_bytes` lowers it."""
        from . import vae_engine as ve
        if not barriers or not in_bboxes:
            return None
        held, resident, reserve, budget = self._residency(ex.program, backend, z.shape[0], in_bboxes, barriers, self._free_bytes(z.device))
        self.last_park_stats.update(budget=budget, reserve=reserve)
        n = len(in_bboxes)
        orders = [list(range(n)) if r % 2 == 0 else list(range(n - 1, -1, -1)) for r in range(len(barriers))]
        parked = ve.plan_residency(orders, resident, budget)
        if not any(parked):
            return None
        sizes = {}       # a tile's buffer: its largest footprint over the barriers where it is parked
        for r, p in enumerate(parked):
            for i in p:
                sizes[i] = max(sizes.get(i, 0), held[r][i])
        ve.require_host_memory(sum(sizes.values()))
        return parked, sizes

    @staticmethod
    def _free_bytes(dev) -> int:
        """Free device memory: the driver's, plus the caching allocator's unused blocks."""
        return torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)

    def _residency(self, program, backend, images, in_bboxes, barriers, free):
        """Bytes the tiles of a pass over `images` images move (held) and keep (resident) at each barrier, the working
        reserve (the largest working set of one tile and two tiles' parked bytes: one upload and one write-back in
        flight) and the budget for the resident tiles: free less the reserve, lowered by `max_resident_bytes`."""
        from . import vae_engine as ve
        fps = {}
        for b in in_bboxes:
            key = (b[3] - b[2], b[1] - b[0])
            if key not in fps:
                fps[key] = ve.tile_footprint(program, backend.name, backend.dtype, key[0], key[1], images, images=images)
        tiles = [fps[(b[3] - b[2], b[1] - b[0])] for b in in_bboxes]
        held = [[fp.held(op.site) for fp in tiles] for op in barriers]            # what a park / upload moves
        resident = [[fp.resident(op.site) for fp in tiles] for op in barriers]    # what a waiting tile holds
        reserve = max(fp.working for fp in fps.values()) + 2 * max((max(h) for h in held), default=0)
        budget = max(free - reserve, 0)
        if self.max_resident_bytes is not None:
            budget = min(budget, max(int(self.max_resident_bytes), 0))
        return held, resident, reserve, budget

    def _images_per_pass(self, program, backend, z, in_bboxes) -> int:
        """How many images of the batch z go through the tensor-core tiles together: `images_per_pass` when set, else
        the largest k whose pass fits in GPU memory (working reserve within the free memory) with no tile parked at any
        barrier under the budget `_park_plan` would use.  1 (a pass per image) when no k > 1 does.  Under the tile
        shard every rank takes the smallest rank's choice, so the statistics rounds pair up."""
        from . import vae_engine as ve
        N = z.shape[0]
        if self.images_per_pass is not None:
            k = max(1, min(int(self.images_per_pass), N))
        else:
            if self.fast_mode:
                _, end = ve.estimated_ops(program, self.color_fix)
                barriers = [op for i, op in enumerate(program.ops) if isinstance(op, ve.Norm) and i >= end]
            else:
                barriers = [op for op in program.ops if isinstance(op, ve.Norm)]
            free = self._free_bytes(z.device)
            n = len(in_bboxes)
            orders = [list(range(n)) if r % 2 == 0 else list(range(n - 1, -1, -1)) for r in range(len(barriers))]

            def fits(k):
                if not in_bboxes:
                    return True
                _, resident, reserve, budget = self._residency(program, backend, k, in_bboxes, barriers, free)
                if reserve > free or any(sum(r) > budget for r in resident):
                    return False
                return not any(ve.plan_residency(orders, resident, budget))
            k = pick_images_per_pass(N, fits)
        if self._shard_world > 1:
            import torch.distributed as dist
            t = torch.tensor([k], dtype=torch.int64, device=z.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self._shard_group)
            k = int(t.item())
        return k

    def _exchange_regions(self, result, out_bboxes, exchanged):
        """Tile shard: every rank pasted its own tiles; gather the disjoint output regions (one all-gather of the
        packed regions -- each byte crosses NVLink once; the round-1 all_reduce of the whole canvas moved it twice).
        exchanged: (images, tiles) per pass; rank r owns shard_tiles(tiles, world, r) of those images.  A tile the inpaint
        mask skipped is in no list: every rank holds its fill already."""
        import torch.distributed as dist
        world, rank = self._shard_world, self._shard_rank
        planes = lambda img: len(range(*img.indices(result.shape[0]))) * result.shape[1]
        area = lambda b: (b[1] - b[0]) * (b[3] - b[2])
        owners = [[(img, shard_tiles(tiles, world, r)) for img, tiles in exchanged] for r in range(world)]
        sizes = [sum(planes(img) * area(out_bboxes[i]) for img, own in jobs for i in own) for jobs in owners]
        cap = max(sizes)
        if cap == 0:
            return
        send = torch.zeros(cap, dtype=result.dtype, device=result.device)
        off = 0
        for img, own in owners[rank]:
            for i in own:
                b = out_bboxes[i]
                blk = result[img, :, b[2]:b[3], b[0]:b[1]]
                send[off:off + blk.numel()].view(blk.shape).copy_(blk)
                off += blk.numel()
        recv = torch.empty(world * cap, dtype=result.dtype, device=result.device)
        dist.all_gather_into_tensor(recv, send, group=self._shard_group)
        for r in range(world):
            if r == rank:
                continue
            off = r * cap
            for img, own in owners[r]:
                for i in own:
                    b = out_bboxes[i]
                    dst = result[img, :, b[2]:b[3], b[0]:b[1]]
                    dst.copy_(recv[off:off + dst.numel()].view(dst.shape))
                    off += dst.numel()
