"""Tiled VAE with the reference's surface (scripts/tilevae.py: `VAEHook`, `GroupNormParam`,
`get_var_mean`, `custom_group_norm`, `crop_valid_region`, `build_task_queue`), H100-native
underneath.

What is different from the reference by design (80 GB of HBM, hand-written sm_90a kernels):
  * tiles, residuals and parked activations stay in HBM -- the reference stages every tile
    through host RAM (`.cpu()` at tilevae.py:534,610,641) and re-uploads it each round;
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
from typing import Callable, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import host
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
            m = mean.mean(dim=0)
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

    def summary(self, stat_len: Optional[int] = None, device=None):
        """-> (mean, var) fp32 tensors, or None when no tile contributed anywhere."""
        if not self.sharded:
            if not self.var_list:
                return None
            var, mean = torch.vstack(self.var_list), torch.vstack(self.mean_list)
            px = torch.tensor(self.pixel_list, dtype=torch.float32, device=var.device)
            px = (px / px.sum()).unsqueeze(1)
            return torch.sum(mean * px, dim=0), torch.sum(var * px, dim=0)
        import torch.distributed as dist
        if self.var_list:
            px = torch.tensor(self.pixel_list, dtype=torch.float32, device=self.var_list[0].device).unsqueeze(1)
            packed = torch.cat([(torch.vstack(self.var_list) * px).sum(0), (torch.vstack(self.mean_list) * px).sum(0), px.sum().view(1)])
        else:
            packed = torch.zeros(2 * int(stat_len) + 1, dtype=torch.float32, device=device)
        dist.all_reduce(packed, group=self.group)
        k = (packed.numel() - 1) // 2
        return packed[k:2 * k] / packed[-1], packed[:k] / packed[-1]


# --------------------------------------------------------------------------- the hook
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

    def __call__(self, x):
        original_device = next(self.net.parameters()).device
        try:
            if self.to_gpu:
                self.net = self.net.to(host.device())
            B, C, H, W = x.shape
            if max(H, W) <= self.pad * 2 + self.tile_size:
                if self.verbose:
                    print("[Tiled VAE]: the input size is tiny and unnecessary to tile.")
                return self.net.original_forward(x)
            return self.vae_tile_forward(x)
        finally:
            self.net = self.net.to(original_device)

    def get_best_tile_size(self, lowerbound, upperbound):
        return lib.td_vae_best_tile_size(int(lowerbound), int(upperbound))

    def split_tiles(self, h, w):
        """tilevae.py:405-462 -> (tile_input_bboxes, tile_output_bboxes), each [x1, x2, y1, y2]."""
        n = check(lib.td_vae_split_tiles(int(h), int(w), int(self.tile_size), int(self.pad), int(self.is_decoder), None, None, 0))
        ib = np.empty((n, 4), dtype=np.int32)
        ob = np.empty((n, 4), dtype=np.int32)
        p = ctypes.POINTER(ctypes.c_int32)
        check(lib.td_vae_split_tiles(int(h), int(w), int(self.tile_size), int(self.pad), int(self.is_decoder),
                                     ib.ctypes.data_as(p), ob.ctypes.data_as(p), n))
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
        per_image = isinstance(backend, ve.TensorCoreBackend)     # channels-last kernels take one image at a time
        est_in = fast_mode_estimator_input(z, tile_size) if self.fast_mode else None

        sharded = self._shard_world > 1
        mine = [i for i in range(len(in_bboxes)) if i % self._shard_world == self._shard_rank] if sharded else list(range(len(in_bboxes)))
        out_c = [op for op in program.ops if isinstance(op, ve.Conv)][-1].module.out_channels
        oh, ow = (height * 8, width * 8) if is_decoder else (height // 8, width // 8)
        result = torch.zeros((N, out_c, oh, ow), dtype=dtype, device=device)   # zeros: a partial (interrupted) result reads 0 elsewhere
        finished = 0
        images = [slice(n, n + 1) for n in range(N)] if per_image else [slice(0, N)]
        for img in images:
            ex = ve.Executor(program, backend)
            if est_in is not None:
                ex.estimate(backend.load(est_in[img]), self.color_fix)
            finished += self._run_tiles(ex, backend, z[img], result[img], [in_bboxes[i] for i in mine], [out_bboxes[i] for i in mine])
            if host.interrupted():
                break
        interrupted = host.interrupted()
        if sharded:
            self._exchange_regions(result, in_bboxes, out_bboxes)
        total = len(mine) * len(images)
        if finished == 0 and total > 0 and interrupted:
            return self._cheap_fallback(z, device, dtype)
        if not interrupted and torch.isnan(result).any():
            raise RuntimeError("[Tiled VAE]: NaN in the result (the reference's test_for_nans, tilevae.py:625)")
        return result

    def _run_tiles(self, ex, backend, z, result, in_bboxes, out_bboxes) -> int:
        """All tiles of one image (or image batch) through the program: rounds separated by the barrier sites."""
        from . import vae_engine as ve
        states = []
        for b in in_bboxes:
            st = ve.TileState(backend.load(z[:, :, b[2]:b[3], b[0]:b[1]]))
            states.append(st)
        sharded = self._shard_world > 1
        rounds = ex.barrier_sites()
        num_tiles = len(states)
        done = 0
        forward = True
        for rnd in range(rounds + 1):
            if host.interrupted():
                break
            collect = GroupNormParam(self._shard_group, sharded)
            site = None
            order = range(num_tiles) if forward else range(num_tiles - 1, -1, -1)     # the reference's zig-zag (:599)
            for i in order:
                if host.interrupted():
                    break
                st = states[i]
                if st is None:
                    continue
                stop = ex.run(st)
                if stop is None:
                    backend.paste(st.act, result, in_bboxes[i], out_bboxes[i], self.is_decoder)
                    states[i] = None
                    done += 1
                else:
                    site = stop
                    var, mean = backend.stats(st.act)
                    collect.add(var, mean, backend.pixels(st.act))
            forward = not forward
            if rnd == rounds or host.interrupted():
                break
            if site is None and sharded:      # a rank without tiles still joins the round's all-reduce
                site = [op for op in ex.program.ops if isinstance(op, ve.Norm) and ex.frozen[op.site] is None][rnd]
            if site is None:
                break
            stat_len = NUM_GROUPS * (z.shape[0] if not isinstance(backend, ve.TensorCoreBackend) else 1)
            merged = collect.summary(stat_len, z.device)
            if merged is None:
                break
            mean, var = merged
            for st in states:
                if st is not None:
                    ex.apply_barrier(st, site, mean, var)
        return done

    def _exchange_regions(self, result, in_bboxes, out_bboxes):
        """Tile shard: every rank pasted its own tiles; gather the disjoint output regions (one all-gather of the
        packed regions -- each byte crosses NVLink once; the round-1 all_reduce of the whole canvas moved it twice)."""
        import torch.distributed as dist
        world, rank = self._shard_world, self._shard_rank
        owners = [[i for i in range(len(out_bboxes)) if i % world == r] for r in range(world)]
        sizes = [sum((out_bboxes[i][1] - out_bboxes[i][0]) * (out_bboxes[i][3] - out_bboxes[i][2]) for i in own) for own in owners]
        plane = result.shape[0] * result.shape[1]
        cap = max(sizes) * plane
        send = torch.zeros(cap, dtype=result.dtype, device=result.device)
        off = 0
        for i in owners[rank]:
            b = out_bboxes[i]
            blk = result[:, :, b[2]:b[3], b[0]:b[1]]
            send[off:off + blk.numel()].view(blk.shape).copy_(blk)
            off += blk.numel()
        recv = torch.empty(world * cap, dtype=result.dtype, device=result.device)
        dist.all_gather_into_tensor(recv, send, group=self._shard_group)
        for r in range(world):
            if r == rank:
                continue
            off = r * cap
            for i in owners[r]:
                b = out_bboxes[i]
                dst = result[:, :, b[2]:b[3], b[0]:b[1]]
                dst.copy_(recv[off:off + dst.numel()].view(dst.shape))
                off += dst.numel()
