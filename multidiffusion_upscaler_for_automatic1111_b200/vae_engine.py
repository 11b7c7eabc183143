"""Tiled-VAE execution engine: the Encoder / Decoder as a compiled op program, run tile by tile.

What the reference does (scripts/tilevae.py:107-204, :464-505, :585-652) -- flatten the ldm network into a task list,
stop every tile at each GroupNorm, merge the tiles' statistics, continue -- is kept as BEHAVIOUR; the machinery is new:

  * `compile_program(net, is_decoder)` walks the module tree once (attribute names of SURVEY section 8(b)) and emits
    typed ops: Conv / Norm / Skip / Attention / Tanh.  Residual adds are not ops: a Conv or Attention op carries
    `add_skip` and the backend fuses the add into its epilogue.  The SiLU after a GroupNorm is a flag of the Norm op.
  * GroupNorm sites are numbered.  A site with frozen statistics (fast mode: measured on the down-sampled input by
    `Executor.estimate`) is applied on the fly; a site without is a barrier: every tile stops there, the per-tile
    statistics are merged (pixel-weighted average of variances and means, the reference's rule) and the round resumes.
  * two backends execute the same program:
      - `TensorCoreBackend` (fp16 / bf16 networks): activations channels-last in HBM, every convolution and the four
        attention GEMMs on wgmma (csrc/td_conv.cu), GroupNorm statistics / apply+SiLU / upsample / softmax on the
        channels-last streaming kernels (csrc/td_nhwc.cu);
      - `ModuleBackend` (fp32 networks or layouts the kernels do not cover): the host application's modules for the
        dense ops, NCHW GroupNorm kernels (csrc/td_vae.cu).
"""
from __future__ import annotations

import os

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from . import vae_ops as ops

NUM_GROUPS = 32
GN_EPS = 1e-6


# ----------------------------------------------------------------------------------------------- program
@dataclass
class Conv:
    module: torch.nn.Module          # nn.Conv2d
    add_skip: bool = False           # out = conv(x) + skip (the ResnetBlock's `x + h`)
    upsample_first: bool = False     # ldm Upsample: nearest x2, then this conv
    downsample: bool = False         # ldm Downsample: pad (0,1,0,1), 3x3 stride 2, no conv padding


@dataclass
class Skip:
    module: Optional[torch.nn.Module] = None   # None: identity shortcut; else nin_shortcut / conv_shortcut of the input


@dataclass
class Norm:
    module: torch.nn.Module          # nn.GroupNorm(32, C, eps=1e-6)
    act: bool                        # SiLU follows
    site: int = -1


@dataclass
class Attention:
    module: torch.nn.Module          # AttnBlock: q, k, v, proj_out (1x1 convs)
    add_skip: bool = True


@dataclass
class Tanh:
    pass


@dataclass
class Program:
    ops: List[object]
    num_sites: int
    is_decoder: bool
    first_resample: int              # index of the first down-sampling op (color-fix cut), or len(ops)
    cache: Dict[str, object] = field(default_factory=dict)    # backend-owned prepared weights


def _res_block(ops_: List[object], block) -> None:
    changes = block.in_channels != block.out_channels
    shortcut = (block.conv_shortcut if block.use_conv_shortcut else block.nin_shortcut) if changes else None
    ops_ += [Skip(shortcut), Norm(block.norm1, True), Conv(block.conv1), Norm(block.norm2, True), Conv(block.conv2, add_skip=True)]


def _attn_block(ops_: List[object], attn) -> None:
    ops_ += [Skip(None), Norm(attn.norm, False), Attention(attn)]


def compile_program(net, is_decoder: bool) -> Program:
    """The op sequence of ldm's Encoder / Decoder forward (what tilevae.py:139-195 flattens into its task queue)."""
    seq: List[object] = [Conv(net.conv_in)]

    def middle():
        _res_block(seq, net.mid.block_1)
        _attn_block(seq, net.mid.attn_1)
        _res_block(seq, net.mid.block_2)

    if is_decoder:
        middle()
        for level in range(net.num_resolutions - 1, -1, -1):
            for b in range(net.num_res_blocks + 1):
                _res_block(seq, net.up[level].block[b])
            if level != 0:
                seq.append(Conv(net.up[level].upsample.conv, upsample_first=True))
    else:
        for level in range(net.num_resolutions):
            for b in range(net.num_res_blocks):
                _res_block(seq, net.down[level].block[b])
            if level != net.num_resolutions - 1:
                seq.append(Conv(net.down[level].downsample.conv, downsample=True))
        middle()
    if not is_decoder or not net.give_pre_end:
        seq += [Norm(net.norm_out, True), Conv(net.conv_out)]
        if is_decoder and net.tanh_out:
            seq.append(Tanh())
    sites = 0
    first_resample = len(seq)
    for i, op in enumerate(seq):
        if isinstance(op, Norm):
            op.site = sites
            sites += 1
        if isinstance(op, Conv) and op.downsample and first_resample == len(seq):
            first_resample = i
    return Program(seq, sites, is_decoder, first_resample)


# ----------------------------------------------------------------------------------------------- residency plan
@dataclass
class TileFootprint:
    """What one tile holds in HBM along the program, in the backend's real layouts.  Per GroupNorm site: `act`, the
    bytes of the activation entering the norm, and `skip`, the bytes of the held shortcut (0 when there is none or
    when it IS the activation: an identity shortcut is one tensor).  `working`: the largest set of live tensors of
    the tile between two sites (its own state, the op's outputs and temporaries, the four-GEMM attention's score
    matrix).  `alias[site]`: the shortcut is the activation (identity shortcut)."""
    act: List[int]
    skip: List[int]
    alias: List[bool]
    working: int

    def held(self, site: int) -> int:
        """Bytes at the site: what parking copies."""
        return self.act[site] + self.skip[site]

    def resident(self, site: int) -> int:
        """Bytes once the site's norm is applied: the normalised activation no longer aliases an identity shortcut."""
        return self.act[site] + (self.act[site] if self.alias[site] else self.skip[site])


def tile_footprint(program: Program, backend_name: str, dtype, h: int, w: int, batch: int = 1,
                   images: Optional[int] = None) -> TileFootprint:
    """Shape walk of `program` for an input tile of h x w pixels.  backend_name "wgmma": channels-last, `images` images
    per pass (None: one), conv_in's input padded to 64 channels, output channels rounded up to 16; "modules": NCHW,
    `batch` images, exact channels."""
    e = torch.empty((), dtype=dtype).element_size()
    tc = backend_name == TensorCoreBackend.name
    n = (images or 1) if tc else batch

    def nbytes(c, hh, ww):
        return n * c * hh * ww * e

    def out_c(m):
        co = m.out_channels
        return (co if co % 16 == 0 else ops.round_up(co, 16)) if tc else co

    c = program.ops[0].module.in_channels
    c = ops.round_up(c, 64) if tc else c
    H, W = h, w
    act, skip, alias = nbytes(c, H, W), 0, False
    act_at: List[int] = []
    skip_at: List[int] = []
    alias_at: List[bool] = []
    working = act

    def live(*extra):
        nonlocal working
        working = max(working, act + (0 if alias else skip) + sum(extra))

    for op in program.ops:
        if isinstance(op, Conv):
            m, tmp = op.module, 0
            if op.upsample_first:
                folded = tc and FOLD_UPSAMPLE and m.kernel_size == (3, 3) and m.out_channels % 16 == 0
                if not folded:
                    tmp = nbytes(c, 2 * H, 2 * W)
                H, W = 2 * H, 2 * W
            if op.downsample:
                if not tc:
                    tmp = nbytes(c, H + 1, W + 1)          # F.pad
                H, W = (H - 2) // 2 + 1, (W - 2) // 2 + 1
            c = out_c(m)
            y = nbytes(c, H, W)
            live(tmp, y, y if tc else 0)                   # tensor cores: a dual-output epilogue writes two
            act, alias = y, False
            if op.add_skip:
                skip = 0
        elif isinstance(op, Skip):
            if op.module is None:
                skip, alias = act, True
            else:
                y = nbytes(out_c(op.module), H, W)
                live(y)
                skip, alias = y, False
        elif isinstance(op, Norm):
            act_at.append(act)
            skip_at.append(0 if alias else skip)
            alias_at.append(alias)
            live(act)
            alias = False
        elif isinstance(op, Attention):
            T = H * W
            y = nbytes(c, H, W)
            if tc:
                qk = 2 * n * T * ops.round_up(c, 8) * e
                if T > SCORE_MATRIX_MAX_TOKENS:
                    extra = qk + 2 * n * T * c * e                              # v, o
                else:                                                           # one image's v^T and scores at a time
                    Tp = ops.round_up(T, 8)
                    extra = qk + c * Tp * e + T * Tp * e + n * T * ops.round_up(c, 8) * e   # v^T, scores, o
                live(extra, y, y)
            else:
                live(3 * y, 2 * y, y)                      # q, k, v; the attention output and its NCHW copy
            act, skip, alias = y, 0, False
        elif isinstance(op, Tanh):
            live(act)
    return TileFootprint(act_at, skip_at, alias_at, working)


def plan_residency(orders: List[List[int]], held: List[List[int]], budget: int) -> List[List[int]]:
    """Which tiles wait in host memory at each barrier.  orders[r]: the tiles in the order round r visits them (round r
    ends at barrier r); held[r][i]: bytes tile i holds in HBM while it waits at barrier r (`TileFootprint.resident`:
    its barrier norm is applied before the next round).  -> parked[r], the tiles parked at barrier r.

    Round r+1 visits the tiles in reverse (the zig-zag), so the tiles visited last in round r are needed first: keep
    the longest suffix of round r's order resident (Belady: what is needed soonest stays).  The suffix is shortened
    until the resident bytes fit the budget at the barrier AND at every point of the round, where the tiles still
    waiting at barrier r-1 and the ones already resident at barrier r are held together."""
    parked: List[List[int]] = []
    prev: Dict[int, int] = {}              # tile -> bytes, resident at the previous barrier
    for r, order in enumerate(orders):
        n = len(order)
        waiting = [0] * (n + 1)           # waiting[k]: bytes of previous residents visited at position >= k
        for k in range(n - 1, -1, -1):
            waiting[k] = waiting[k + 1] + prev.get(order[k], 0)
        keep = n
        while keep > 0:
            first = n - keep
            kept, ok = 0, True
            for k in range(n + 1):         # after k visits
                if k > first:
                    kept += held[r][order[k - 1]]
                if kept + waiting[k] > budget:
                    ok = False
                    break
            if ok:
                break
            keep -= 1
        resident = order[n - keep:]
        parked.append(order[:n - keep])
        prev = {t: held[r][t] for t in resident}
    return parked


def host_available_bytes(meminfo: str = "/proc/meminfo", cgroup: str = "/sys/fs/cgroup") -> Optional[int]:
    """MemAvailable of the host, lowered to what the process's cgroup (v2) still allows when it has a memory limit (a
    container's cap is not in /proc/meminfo); None where neither is reported."""
    avail = None
    try:
        with open(meminfo) as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    avail = int(line.split()[1]) * 1024
                    break
    except OSError:
        pass
    try:
        with open(os.path.join(cgroup, "memory.max")) as f:
            cap = f.read().strip()
        with open(os.path.join(cgroup, "memory.current")) as f:
            used = int(f.read().strip())
        if cap != "max":
            left = max(int(cap) - used, 0)
            avail = left if avail is None else min(avail, left)
    except (OSError, ValueError):
        pass
    return avail


def require_host_memory(need: int, available: Optional[int] = None) -> None:
    """Refuse a parking plan the host cannot pin, before any tile runs (rather than letting the OOM killer decide)."""
    if available is None:
        available = host_available_bytes()
    if available is not None and need > available:
        raise RuntimeError(f"[Tiled VAE]: parking the tiles that do not fit in GPU memory needs {need / 1e9:.1f} GB of pinned "
                           f"host memory, but only {available / 1e9:.1f} GB are available; use a smaller image or a "
                           f"smaller tile size, or free host memory")


# ----------------------------------------------------------------------------------------------- backends
def _f32(t: Optional[torch.Tensor], device) -> Optional[torch.Tensor]:
    return None if t is None else t.detach().to(device=device, dtype=torch.float32).contiguous()


def _periodic_pieces(lo: int, hi: int, L: int):
    """[lo, hi) in unwrapped coordinates as (offset in the span, start in [0, L), length) pieces that stay inside one period."""
    out, p = [], lo
    while p < hi:
        s = p % L
        n = min(hi - p, L - s)
        out.append((p - lo, s, n))
        p += n
    return out


class ModuleBackend:
    """NCHW activations; dense ops through the host application's modules, GroupNorm through csrc/td_vae.cu."""
    name = "modules"

    def __init__(self, program: Program, device, dtype):
        self.program, self.device, self.dtype = program, device, dtype
        self._affine = program.cache.setdefault("module_affine", {})

    def load(self, z_view: torch.Tensor) -> torch.Tensor:
        from .tilevae import copy_region
        t = torch.empty(z_view.shape, dtype=self.dtype, device=self.device)
        copy_region(z_view, t)
        return t

    def load_wrap(self, z: torch.Tensor, bbox) -> torch.Tensor:
        """Tile [x1, x2) x [y1, y2) of the periodic canvas z, bounds in unwrapped coordinates: one td_copy_region per piece
        of the tile that lies in one period (four when the tile straddles both seams)."""
        from .tilevae import copy_region
        x1, x2, y1, y2 = (int(v) for v in bbox)
        H, W = z.shape[2], z.shape[3]
        t = torch.empty((z.shape[0], z.shape[1], y2 - y1, x2 - x1), dtype=self.dtype, device=self.device)
        for ty0, sy0, ny in _periodic_pieces(y1, y2, H):
            for tx0, sx0, nx in _periodic_pieces(x1, x2, W):
                copy_region(z[:, :, sy0:sy0 + ny, sx0:sx0 + nx], t[:, :, ty0:ty0 + ny, tx0:tx0 + nx])
        return t

    def pixels(self, a: torch.Tensor) -> int:
        return a.shape[2] * a.shape[3]

    def conv(self, a, op: Conv, skip):
        if op.upsample_first:
            a = F.interpolate(a, scale_factor=2.0, mode="nearest")
        if op.downsample:
            a = F.pad(a, (0, 1, 0, 1), mode="constant", value=0)
        y = op.module(a)
        return y.add_(skip) if skip is not None else y

    def shortcut(self, a, op: Skip):
        return a if op.module is None else op.module(a)

    def stats(self, a):
        from .tilevae import get_var_mean
        return get_var_mean(a, NUM_GROUPS)

    def norm(self, a, op: Norm, mean, var):
        from .tilevae import custom_group_norm
        key = id(op.module)
        if key not in self._affine:
            self._affine[key] = (_f32(getattr(op.module, "weight", None), self.device), _f32(getattr(op.module, "bias", None), self.device))
        gamma, beta = self._affine[key]
        return custom_group_norm(a, NUM_GROUPS, mean, var, gamma, beta, GN_EPS, act=op.act)

    def attention(self, a, op: Attention, skip):
        m = op.module
        q, k, v = m.q(a), m.k(a), m.v(a)
        b, c, h, w = q.shape
        q, k, v = (t.reshape(b, 1, c, h * w).transpose(2, 3) for t in (q, k, v))
        o = F.scaled_dot_product_attention(q, k, v)                      # softmax(q k^T / sqrt(c)) v, tile_utils/attn.py:49-72
        y = m.proj_out(o.transpose(2, 3).reshape(b, c, h, w))
        return y.add_(skip) if skip is not None else y

    def tanh(self, a):
        return torch.tanh(a)

    def has_nan(self, a) -> torch.Tensor:
        return torch.isnan(a).any()

    def out_channels(self, a) -> int:
        return a.shape[1]

    def paste(self, a, result, in_bbox, out_bbox, is_decoder: bool):
        from .tilevae import copy_region, crop_valid_region
        valid = crop_valid_region(a.to(result.dtype).contiguous(), in_bbox, out_bbox, is_decoder)
        copy_region(valid, result[:, :, out_bbox[2]:out_bbox[3], out_bbox[0]:out_bbox[1]])


FOLD_UPSAMPLE = os.environ.get("TD_VAE_FOLD_UPSAMPLE", "1") != "0"     # 0: materialise the upsampled tensor (measurement only)
DUAL_OUTPUT = os.environ.get("TD_VAE_DUAL_OUTPUT", "1") != "0"         # 0: separate GroupNorm pass at block boundaries (measurement only)
# Attention tiles with more tokens than this run the fused kernel (vae_ops.attention): 46340 = floor(sqrt(2^31)), so
# their [T, T] score matrix would pass 2^31 elements (4 GiB in fp16), and the reference's H100 default tiles (decoder
# 256, encoder 3072) need 11-27 GiB of it.  Smaller tiles keep the four-GEMM path and its exact output.  That path
# allocates the scores as [T, Tp], Tp = round_up(T, 8), so its largest matrix (T = 46340: 46340 x 46344 =
# 2^31 + 97312 elements) does pass 2^31 elements; the score GEMM, softmax_rows and the P V GEMM address it with 64-bit
# offsets (tests/test_gpu_vae_large_tiles.py checks that tile).  The bound depends only on the tile, so a tile takes the
# same path, with the same bits, on any card.
SCORE_MATRIX_MAX_TOKENS = 46340


class TensorCoreBackend:
    """Channels-last activations; convolutions and attention GEMMs on wgmma, the rest on streaming kernels."""
    name = "wgmma"

    def __init__(self, program: Program, device, dtype):
        self.program, self.device, self.dtype = program, device, dtype
        self._w = program.cache.setdefault(f"tc_weights_{dtype}", {})

    # ---- prepared weights (once per network and dtype) -------------------------------------------------------
    def _conv_w(self, conv: torch.nn.Module):
        key = id(conv)
        if key not in self._w:
            co, ci, kh, kw = conv.weight.shape
            cout_rows = co if co % 16 == 0 else ops.round_up(co, 16)
            wp = ops.pack_conv_weight(conv.weight.to(self.device), self.dtype, cin_pad=ops.round_up(ci, 64), cout_pad=cout_rows)
            b = torch.zeros(cout_rows, dtype=torch.float32, device=self.device)
            if conv.bias is not None:
                b[:co] = conv.bias.detach().float()
            self._w[key] = (wp, b, co, cout_rows, kh)
        return self._w[key]

    def _upconv_w(self, conv: torch.nn.Module):
        """Folded taps of a 3x3 convolution behind a nearest-2x upsample (td_upconv2x_nhwc)."""
        key = ("up2", id(conv))
        if key not in self._w:
            ci = conv.weight.shape[1]
            self._w[key] = ops.fold_upsample_weight(conv.weight.to(self.device), self.dtype, cin_pad=ops.round_up(ci, 64))
        return self._w[key]

    def _affine(self, norm: torch.nn.Module):
        key = id(norm)
        if key not in self._w:
            self._w[key] = (_f32(getattr(norm, "weight", None), self.device), _f32(getattr(norm, "bias", None), self.device))
        return self._w[key]

    @staticmethod
    def supports(program: Program, dtype) -> bool:
        if dtype not in (torch.float16, torch.bfloat16):
            return False
        for op in program.ops:
            if isinstance(op, Conv):
                m = op.module
                if not isinstance(m, torch.nn.Conv2d) or m.kernel_size not in ((1, 1), (3, 3)) or m.groups != 1 or m.dilation != (1, 1):
                    return False
                if op.downsample and (m.stride != (2, 2) or m.padding != (0, 0)):
                    return False
                if not op.downsample and (m.stride != (1, 1) or m.padding != (m.kernel_size[0] // 2,) * 2):
                    return False
            if isinstance(op, Norm):
                c = op.module.num_channels
                if op.module.num_groups != NUM_GROUPS or c % 128 != 0 or 256 % (c // 8) != 0:
                    return False
            if isinstance(op, Skip) and op.module is not None and not isinstance(op.module, torch.nn.Conv2d):
                return False
        return True

    # ---- ops --------------------------------------------------------------------------------------------------
    def load(self, z_view: torch.Tensor) -> torch.Tensor:
        return ops.nchw_to_nhwc(z_view.to(self.dtype) if z_view.dtype != self.dtype else z_view, ops.round_up(z_view.shape[1], 64))

    def load_wrap(self, z: torch.Tensor, bbox) -> torch.Tensor:
        """Tile [x1, x2) x [y1, y2) of the periodic canvas z (bounds in unwrapped coordinates): one modular gather with the
        layout change and channel padding of `load`."""
        z = z.to(self.dtype) if z.dtype != self.dtype else z
        return ops.nchw_to_nhwc_wrap(z.contiguous(), bbox, ops.round_up(z.shape[1], 64))

    def pixels(self, a) -> int:
        return a.shape[1] * a.shape[2]

    fuses_norm = True      # conv(..., post=...) applies a following frozen GroupNorm (+ SiLU) in the epilogue

    def conv(self, a, op: Conv, skip, post=None, dual=False):
        """post: the frozen GroupNorm (+ SiLU) that follows, applied in the epilogue; dual: return (raw, normalised)."""
        wp, b, co, cout_rows, k = self._conv_w(op.module)
        if op.upsample_first:
            if k == 3 and skip is None and cout_rows == co and FOLD_UPSAMPLE:
                # ldm Upsample block: the four parity convolutions of the low-resolution tile, no 4x intermediate
                return ops.upconv2x_nhwc(a, self._upconv_w(op.module), b, cout=cout_rows, post=post, dual=dual)
            a = ops.upsample2x_nhwc(a)
        _, H, W, _ = a.shape
        if op.downsample:
            oh, ow = (H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1
            return ops.conv2d_nhwc(a, wp, b, ksize=3, stride=2, pad=(0, 0), out_hw=(oh, ow), residual=skip, cout=cout_rows, post=post, dual=dual)
        return ops.conv2d_nhwc(a, wp, b, ksize=k, pad=(k // 2, k // 2), residual=skip, cout=cout_rows, post=post, dual=dual)

    def norm_affine(self, op: Norm, mean, var):
        """Per-image, per-channel (scale [n, C], shift [n, C], act) equivalent to custom_group_norm (+ SiLU) with the
        statistics mean / var [n * groups]: y = x * gamma[c] / sqrt(var[g] + eps) + (beta[c] - mean[g] * gamma[c] /
        sqrt(var[g] + eps)).  Element-wise, so an image's constants do not depend on the other images."""
        gamma, beta = self._affine(op.module)
        c = op.module.num_channels
        cpg = c // NUM_GROUPS
        rstd = (1.0 / torch.sqrt(var.float().view(-1, NUM_GROUPS) + GN_EPS)).repeat_interleave(cpg, dim=1)
        scale = rstd * gamma if gamma is not None else rstd
        shift = -mean.float().view(-1, NUM_GROUPS).repeat_interleave(cpg, dim=1) * scale
        if beta is not None:
            shift = shift + beta
        return scale.contiguous(), shift.contiguous(), bool(op.act)

    def shortcut(self, a, op: Skip):
        if op.module is None:
            return a
        wp, b, co, cout_rows, k = self._conv_w(op.module)
        return ops.conv2d_nhwc(a, wp, b, ksize=k, pad=(k // 2, k // 2), cout=cout_rows)

    def stats(self, a):
        return ops.gn_stats_nhwc(a, NUM_GROUPS)

    def norm(self, a, op: Norm, mean, var):
        gamma, beta = self._affine(op.module)
        return ops.gn_apply_nhwc(a, mean, var, gamma, beta, op.act, NUM_GROUPS, GN_EPS)

    def attention(self, a, op: Attention, skip, post=None, dual=False):
        """softmax(q k^T / sqrt(C)) v + proj_out (tile_utils/attn.py:49-72) of each of the n images of a [n, H, W, C]
        tile.  The q / k / v projections of all images are one GEMM (a row's result does not depend on its neighbours).
        Up to SCORE_MATRIX_MAX_TOKENS tokens: per image, the scores, one row softmax and the P V GEMM, the [tokens, tokens]
        score matrix in HBM (388 MB fp16 for a 118 x 118 tile); larger tiles: the fused online-softmax kernel over all
        images in one launch, no score matrix."""
        m = op.module
        n, H, W, C = a.shape
        T = H * W
        x2 = a.view(n * T, C)
        wq, bq, *_ = self._conv_w(m.q)
        wk, bk, *_ = self._conv_w(m.k)
        wv, bv, *_ = self._conv_w(m.v)
        q = ops.gemm_nt(x2, wq[0], bias=bq)
        k = ops.gemm_nt(x2, wk[0], bias=bk)
        wp, bp, *_ = self._conv_w(m.proj_out)
        alpha = float(int(C) ** -0.5)
        if T > SCORE_MATRIX_MAX_TOKENS:
            v = ops.gemm_nt(x2, wv[0], bias=bv)
            per = (lambda t: t) if n == 1 else (lambda t: t.unflatten(0, (n, T)))     # [T, C] for one image, [n, T, C] for several
            o = ops.attention(per(q), per(k), per(v), alpha)
            return ops.conv2d_nhwc(o.view(n, H, W, C), wp, bp, ksize=1, residual=skip, post=post, dual=dual)
        Tp = ops.round_up(T, 8)
        o = torch.empty((n * T, C), dtype=self.dtype, device=self.device)
        for i in range(n):
            rows = slice(i * T, (i + 1) * T)
            vt = torch.empty((C, Tp), dtype=self.dtype, device=self.device)
            if Tp != T:
                vt[:, T:].zero_()      # K of the P V GEMM runs over the padded pitch: P's padding is 0, V's must be finite
            # V^T[c, t] = sum_i Wv[c, i] x[t, i] + bv[c]: the GEMM with the operands swapped, bias per output row
            ops.gemm_nt(wv[0], x2[rows], bias=bv, bias_per_row=True, out=vt[:, :T])
            s = torch.empty((T, Tp), dtype=self.dtype, device=self.device)
            ops.gemm_nt(q[rows], k[rows], alpha=alpha, out=s[:, :T])
            ops.softmax_rows(s, T, out=s)
            ops.gemm_nt(s, vt, out=o[rows])    # K = Tp (a multiple of 8; the last partial 64-chunk is zero-filled by the TMA unit)
            del vt, s                  # one image's scores at a time
        return ops.conv2d_nhwc(o.view(n, H, W, C), wp, bp, ksize=1, residual=skip, post=post, dual=dual)

    def tanh(self, a):
        return torch.tanh(a)

    def has_nan(self, a) -> torch.Tensor:
        return torch.isnan(a).any()

    def out_channels(self, a) -> int:
        last = [op for op in self.program.ops if isinstance(op, Conv)][-1]
        return last.module.out_channels

    def paste(self, a, result, in_bbox, out_bbox, is_decoder: bool):
        padded = [v * 8 if is_decoder else v // 8 for v in in_bbox]
        m = [out_bbox[i] - padded[i] for i in range(4)]
        _, H, W, _ = a.shape
        src = a[:, m[2]:H + m[3], m[0]:W + m[1], :]
        c = result.shape[1]
        ops.nhwc_to_nchw_region(src, result[:, :, out_bbox[2]:out_bbox[3], out_bbox[0]:out_bbox[1]], c)


def pick_backend(program: Program, device, dtype):
    if TensorCoreBackend.supports(program, dtype):
        return TensorCoreBackend(program, device, dtype)
    return ModuleBackend(program, device, dtype)


# ----------------------------------------------------------------------------------------------- executor
def estimated_ops(program: Program, color_fix: bool) -> Tuple[int, int]:
    """(index of the last Norm op, end of the ops `Executor.estimate` runs): fast mode freezes the sites of the Norm ops
    before `end`; the others stay barriers."""
    last_norm = max(i for i, op in enumerate(program.ops) if isinstance(op, Norm))
    return last_norm, min(last_norm + 1, program.first_resample if color_fix else len(program.ops))


@dataclass
class TileState:
    act: object
    skip: object = None
    pc: int = 0
    pixels: int = 0


class Executor:
    """Runs a Program over tiles.  `frozen[site]` = (mean, var) applied on the fly, or None = barrier site."""

    def __init__(self, program: Program, backend):
        self.program, self.be = program, backend
        self.frozen: List[Optional[Tuple[torch.Tensor, torch.Tensor]]] = [None] * program.num_sites
        self._affine_cache: Dict[int, tuple] = {}

    def _step(self, st: TileState, op) -> None:
        be = self.be
        if isinstance(op, Skip):
            st.skip = be.shortcut(st.act, op)
        elif isinstance(op, Conv):
            st.act = be.conv(st.act, op, st.skip if op.add_skip else None)
            if op.add_skip:
                st.skip = None
        elif isinstance(op, Attention):
            st.act = be.attention(st.act, op, st.skip if op.add_skip else None)
            st.skip = None
        elif isinstance(op, Tanh):
            st.act = be.tanh(st.act)
        else:
            raise TypeError(f"unknown op {op!r}")

    def run(self, st: TileState, stop: Optional[int] = None) -> Optional[Norm]:
        """Advance until the next barrier site (returned; st.pc stays ON the Norm op) or the end / `stop` (None)."""
        opsq = self.program.ops
        end = len(opsq) if stop is None else stop
        fuse = getattr(self.be, "fuses_norm", False)
        while st.pc < end:
            op = opsq[st.pc]
            if isinstance(op, Norm):
                fz = self.frozen[op.site]
                if fz is None:
                    return op
                st.act = self.be.norm(st.act, op, fz[0], fz[1])
            elif fuse and DUAL_OUTPUT and isinstance(op, (Conv, Attention)) and st.pc + 2 < end and isinstance(opsq[st.pc + 1], Skip) \
                    and isinstance(opsq[st.pc + 2], Norm) and self.frozen[opsq[st.pc + 2].site] is not None \
                    and self._dual_ok(op, opsq[st.pc + 2]):
                # producer -> [shortcut source] -> GroupNorm (+ SiLU) with frozen statistics (the boundary between two
                # ResnetBlocks / attention): the producer writes BOTH tensors -- the raw one feeds the shortcut, the
                # normalised one is the next block's input; no pass over the activation in between
                skp, nxt = opsq[st.pc + 1], opsq[st.pc + 2]
                if nxt.site not in self._affine_cache:
                    self._affine_cache[nxt.site] = self.be.norm_affine(nxt, *self.frozen[nxt.site])
                fn = self.be.conv if isinstance(op, Conv) else self.be.attention
                raw, normed = fn(st.act, op, st.skip if op.add_skip else None, post=self._affine_cache[nxt.site], dual=True)
                st.skip = self.be.shortcut(raw, skp)
                st.act = normed
                st.pc += 2
            elif fuse and isinstance(op, Conv) and st.pc + 1 < end and isinstance(opsq[st.pc + 1], Norm) \
                    and self.frozen[opsq[st.pc + 1].site] is not None:
                # conv -> GroupNorm (+ SiLU) with frozen statistics: the norm rides in the conv's epilogue (the raw conv
                # output has no other reader: a residual source is always separated from its norm by a Skip op)
                nxt = opsq[st.pc + 1]
                if nxt.site not in self._affine_cache:
                    self._affine_cache[nxt.site] = self.be.norm_affine(nxt, *self.frozen[nxt.site])
                st.act = self.be.conv(st.act, op, st.skip if op.add_skip else None, post=self._affine_cache[nxt.site])
                if op.add_skip:
                    st.skip = None
                st.pc += 1
            else:
                self._step(st, op)
            st.pc += 1
        return None

    @staticmethod
    def _dual_ok(op, norm: Norm) -> bool:
        """The kernel's post stage runs on whole 16-channel groups of real output channels."""
        m = op.module if isinstance(op, Conv) else op.module.proj_out
        return m.out_channels % 16 == 0 and m.out_channels == norm.module.num_channels

    def apply_barrier(self, st: TileState, op: Norm, mean, var) -> None:
        st.act = self.be.norm(st.act, op, mean, var)
        st.pc += 1

    @torch.no_grad()
    def estimate(self, act, color_fix: bool, report: bool = True) -> bool:
        """Fast mode (tilevae.py:464-505): run the program on the down-sampled input, freezing each GroupNorm site
        with the statistics of that single tensor (per image on the tensor cores).  With color_fix the sites from the
        first down-sampling on stay barriers (`estimated_ops`).  Returns False (nothing frozen) when a NaN shows up;
        `report`: say so on stdout."""
        if self.program.num_sites == 0:
            raise ValueError("No group norm found in the task queue")
        opsq = self.program.ops
        last_norm, end = estimated_ops(self.program, color_fix)
        st = TileState(act)
        frozen: List[Optional[Tuple[torch.Tensor, torch.Tensor]]] = [None] * self.program.num_sites
        nan = None
        for i in range(end):
            op = opsq[i]
            if isinstance(op, Norm):
                var, mean = self.be.stats(st.act)
                frozen[op.site] = (mean, var)
                if i == last_norm:
                    break
                st.act = self.be.norm(st.act, op, mean, var)
            else:
                self._step(st, op)
            flag = self.be.has_nan(st.act)
            nan = flag if nan is None else (nan | flag)
        if nan is not None and bool(nan):
            if report:
                print("Nan detected in fast mode estimation. Fast mode disabled.")
            return False
        self.frozen = frozen
        self._affine_cache = {}
        return True

    def barrier_sites(self) -> int:
        return sum(1 for f in self.frozen if f is None)
