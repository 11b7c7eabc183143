"""Tile shard across the GPUs of one box (one process per GPU, `torch.distributed` for the plumbing).

The reference is single-device (SURVEY.md section 5); this is new work behind the same delegate API:
`delegate.init_tile_shard(group, fused=True)` after `init_grid_bbox`.  Rank r scatters and denoises
the contiguous chunk `[r*chunk, (r+1)*chunk)` of the row-major tile list; then either

  * fused (default): the tile outputs are placed in an exchange buffer that every peer has mapped
    through CUDA IPC, `td_peer_signal` publishes the step counter into the peers' flag arrays, and
    `td_blend_multidiffusion_peer` waits for all ranks and blends while reading the peers' tiles over
    NVLink -- one kernel does the "all-gather" and the blend, no NCCL call on the data path;
  * NCCL: `all_gather_into_tensor` of the padded chunks, then the ordinary pointer-table blend.

Either way every rank runs the identical deterministic blend, so the latent is bit-identical on all
ranks and to a single-GPU run.
"""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

from . import _cabi, engine
from ._cabi import check, lib


class TileShard:
    """Contiguous partition of T tiles over `world` ranks (chunk = ceil(T / world))."""

    def __init__(self, num_tiles: int, rank: int, world: int):
        if not (0 <= rank < world):
            raise ValueError(f"rank {rank} outside world {world}")
        self.num_tiles, self.rank, self.world = num_tiles, rank, world
        self.chunk = -(-num_tiles // world)
        self.begin = min(rank * self.chunk, num_tiles)
        self.end = min(self.begin + self.chunk, num_tiles)
        self.num_chunks = -(-num_tiles // self.chunk) if self.chunk else 0    # ranks >= num_chunks own no tile

    @property
    def num_local(self) -> int:
        return self.end - self.begin

    def owner(self, tile: int) -> int:
        return tile // self.chunk


def gather_tile_outputs(local_padded: torch.Tensor, group=None) -> torch.Tensor:
    """all-gather of the per-rank padded chunks -> [world*chunk*N, C, th, tw] (any backend / device)."""
    world = dist.get_world_size(group)
    out = torch.empty((world * local_padded.shape[0],) + tuple(local_padded.shape[1:]), dtype=local_padded.dtype,
                      device=local_padded.device)
    try:
        dist.all_gather_into_tensor(out, local_padded.contiguous(), group=group)
    except (RuntimeError, NotImplementedError):   # backends without the tensor variant
        parts = list(out.chunk(world, dim=0))
        dist.all_gather(parts, local_padded.contiguous(), group=group)
    return out


class RegionShard:
    """Region prompt control under the tile shard (pure bookkeeping, no device work): which rank denoises which custom
    region, and how the region rectangles and outputs are packed for the two all-gathers of a step.

    Region j (list order) is denoised by rank j % world, on every rank the same without any communication.  Every rank
    then needs every region output for the composite (replicate mode: of the whole canvas; strip mode: of its own rows),
    so the owners' outputs are packed back to back in list order, padded to the largest rank's pack and all-gathered.
    In strip mode a rank holds valid latent rows only in its own strip: the rows of region j that lie in strip [B[q],
    B[q+1]) are packed by rank q and reach the owner of j through one more all-gather before the denoiser calls."""

    def __init__(self, rects: Sequence[Sequence[int]], rank: int, world: int):
        if not (0 <= rank < world):
            raise ValueError(f"rank {rank} outside world {world}")
        self.rects = [tuple(int(v) for v in r) for r in rects]        # (x, y, w, h) in latent pixels
        self.rank, self.world = rank, world
        self.owner = [j % world for j in range(len(self.rects))]

    def mine(self, r: Optional[int] = None) -> List[int]:
        """Regions denoised by rank r, in list order."""
        r = self.rank if r is None else r
        return [j for j, o in enumerate(self.owner) if o == r]

    # ---- outputs: owners -> every rank -----------------------------------------------------------------------
    def _area(self, j: int) -> int:
        return self.rects[j][2] * self.rects[j][3]

    def output_pack_numel(self, planes: int) -> int:
        """Elements of one rank's padded output pack (planes = N * C)."""
        return planes * max(sum(self._area(j) for j in self.mine(r)) for r in range(self.world))

    def pack_outputs(self, outs: Sequence[torch.Tensor], planes: int, like: torch.Tensor,
                     dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """This rank's region outputs (in `mine()` order, [N, C, h, w] each) -> one flat padded pack of `dtype` (default:
        like's dtype) on like's device.  The pack must carry the values the denoiser returned -- an fp32 output on an fp16
        latent rounded to fp16 here would be rounded twice by the composite -- so an output is packed only into its own
        dtype or into fp32, which holds every output dtype exactly; anything else is refused."""
        mine = self.mine()
        if len(outs) != len(mine):
            raise ValueError(f"{len(outs)} region outputs for {len(mine)} regions of rank {self.rank}")
        dtype = like.dtype if dtype is None else dtype
        for j, o in zip(mine, outs):
            if o.dtype != dtype and dtype != torch.float32:
                raise ValueError(f"region {j}: a {o.dtype} output does not fit a {dtype} pack exactly")
        pack = torch.zeros(self.output_pack_numel(planes), dtype=dtype, device=like.device)
        off = 0
        for j, o in zip(mine, outs):
            n = planes * self._area(j)
            pack[off:off + n].view(o.shape).copy_(o)
            off += n
        return pack

    def unpack_outputs(self, gathered: torch.Tensor, N: int, C: int) -> List[torch.Tensor]:
        """[world, pack] -> every region's output [N, C, h, w] in list order (views of `gathered`)."""
        outs: List[Optional[torch.Tensor]] = [None] * len(self.rects)
        for r in range(self.world):
            off = 0
            for j in self.mine(r):
                _, _, w, h = self.rects[j]
                n = N * C * w * h
                outs[j] = gathered[r, off:off + n].view(N, C, h, w)
                off += n
        return outs

    # ---- inputs in strip mode: row owners -> region owner ----------------------------------------------------
    def input_pieces(self, lo: int, hi: int) -> List[tuple]:
        """[(region j, a, b)]: the canvas rows [a, b) of region j that lie in [lo, hi), in list order."""
        out = []
        for j, (_, y, _, h) in enumerate(self.rects):
            a, b = max(y, lo), min(y + h, hi)
            if b > a:
                out.append((j, a, b))
        return out

    def input_pack_numel(self, B: Sequence[int], planes: int) -> int:
        return planes * max(sum((b - a) * self.rects[j][2] for j, a, b in self.input_pieces(B[r], B[r + 1])) for r in range(self.world))

    def pack_inputs(self, x: torch.Tensor, B: Sequence[int]) -> torch.Tensor:
        """The rows of every region rectangle inside this rank's strip [B[rank], B[rank+1]) of x [N, C, H, W] -> one flat
        padded pack (only those rows of x are read)."""
        planes = x.shape[0] * x.shape[1]
        pack = torch.zeros(self.input_pack_numel(B, planes), dtype=x.dtype, device=x.device)
        off = 0
        for j, a, b in self.input_pieces(B[self.rank], B[self.rank + 1]):
            rx, _, w, _ = self.rects[j]
            n = planes * (b - a) * w
            pack[off:off + n].view(x.shape[0], x.shape[1], b - a, w).copy_(x[:, :, a:b, rx:rx + w])
            off += n
        return pack

    def unpack_inputs(self, gathered: torch.Tensor, B: Sequence[int], N: int, C: int) -> dict:
        """[world, pack] -> {j: region j's input [N, C, h, w]} for this rank's regions."""
        mine = set(self.mine())
        ins = {}
        for j in mine:
            _, _, w, h = self.rects[j]
            ins[j] = torch.empty((N, C, h, w), dtype=gathered.dtype, device=gathered.device)
        for r in range(self.world):
            off = 0
            for j, a, b in self.input_pieces(B[r], B[r + 1]):
                _, y, w, _ = self.rects[j]
                n = N * C * (b - a) * w
                if j in mine:
                    ins[j][:, :, a - y:b - y] = gathered[r, off:off + n].view(N, C, b - a, w)
                off += n
        return ins


def gather_region_inputs(rs: RegionShard, x: torch.Tensor, B: Sequence[int], group=None) -> dict:
    """Strip mode: one all-gather of the strip-packed region rows -> {j: input of region j} for this rank's regions."""
    N, C = x.shape[0], x.shape[1]
    gathered = gather_tile_outputs(rs.pack_inputs(x, B).view(1, -1), group)
    return rs.unpack_inputs(gathered, B, N, C)


def exchange_region_outputs(rs: RegionShard, outs: Sequence[torch.Tensor], like: torch.Tensor, group=None) -> List[torch.Tensor]:
    """One all-gather of the packed region outputs -> every region's output, in list order, on every rank.  The packs are
    fp32 on every rank: exact for every output dtype, and the same on a rank that owns no region and so cannot know the
    UNet's output dtype, without a collective to agree on one (DESIGN.md section 5)."""
    N, C = like.shape[0], like.shape[1]
    gathered = gather_tile_outputs(rs.pack_outputs(outs, N * C, like, torch.float32).view(1, -1), group)
    return rs.unpack_outputs(gathered, N, C)


class _RawCudaBuffer:
    """A cudaMalloc'd (IPC-exportable) buffer exposed to torch without a copy."""

    def __init__(self, nbytes: int):
        p = ctypes.c_void_p()
        check(lib.td_dev_alloc(int(nbytes), ctypes.byref(p)))
        self.ptr, self.nbytes = p.value, int(nbytes)
        self.__cuda_array_interface__ = {"shape": (self.nbytes,), "typestr": "|u1", "data": (self.ptr, False), "version": 3}

    def tensor(self, device) -> torch.Tensor:
        return torch.as_tensor(self, device=device)

    def handle(self) -> bytes:
        h = ctypes.create_string_buffer(_cabi.TD_IPC_HANDLE_BYTES)
        check(lib.td_ipc_get_handle(ctypes.c_void_p(self.ptr), h))
        return h.raw

    def free(self):
        if self.ptr:
            lib.td_dev_free(ctypes.c_void_p(self.ptr))
            self.ptr = 0


class PeerExchange:
    """Double-buffered tile-output exchange + step flags, mapped into every rank through CUDA IPC."""

    def __init__(self, nbytes: int, device: torch.device, group=None):
        self.group, self.device = group, device
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if self.world > _cabi.TD_MAX_PEERS:
            raise ValueError(f"world size {self.world} exceeds TD_MAX_PEERS={_cabi.TD_MAX_PEERS}")
        self.nbytes = (int(nbytes) + 255) // 256 * 256
        with torch.cuda.device(device):
            self._bufs = [_RawCudaBuffer(self.nbytes), _RawCudaBuffer(self.nbytes)]
            self._flags = _RawCudaBuffer(256)
            torch.cuda.synchronize(device)
            mine = [b.handle() for b in self._bufs] + [self._flags.handle()]
            everyone: List[Optional[list]] = [None] * self.world
            dist.all_gather_object(everyone, mine, group=group)
            self._opened: List[int] = []
            self.buf_ptrs = [[0] * self.world, [0] * self.world]   # [parity][rank] -> device pointer valid HERE
            self.flag_ptrs = [0] * self.world
            for r in range(self.world):
                if r == self.rank:
                    self.buf_ptrs[0][r], self.buf_ptrs[1][r] = self._bufs[0].ptr, self._bufs[1].ptr
                    self.flag_ptrs[r] = self._flags.ptr
                    continue
                ptrs = []
                for h in everyone[r]:
                    p = ctypes.c_void_p()
                    check(lib.td_ipc_open(ctypes.create_string_buffer(h, len(h)), ctypes.byref(p)))
                    ptrs.append(p.value)
                    self._opened.append(p.value)
                self.buf_ptrs[0][r], self.buf_ptrs[1][r], self.flag_ptrs[r] = ptrs
        self._flag_table = (ctypes.c_void_p * self.world)(*self.flag_ptrs)
        self.step = 0
        dist.barrier(group=group)

    def local_buffer(self, parity: int, dtype: torch.dtype) -> torch.Tensor:
        return self._bufs[parity].tensor(self.device).view(dtype)

    @property
    def counter_ptr(self) -> int:
        """This rank's device-side step counter (lives behind the flag slots of the same allocation)."""
        return self._flags.ptr + 128

    def signal(self):
        """Bump the device-side step counter and publish it to every rank (replayable in a CUDA graph)."""
        with torch.cuda.device(self.device):
            check(lib.td_peer_signal(self._flag_table, self.world, self.rank, ctypes.c_void_p(self.counter_ptr),
                                     _cabi.current_stream_ptr(self.device)))

    def close(self):
        for p in self._opened:
            lib.td_ipc_close(ctypes.c_void_p(p))
        self._opened = []
        for b in self._bufs + [self._flags]:
            b.free()


def blend_multidiffusion_peer(g, exchange: PeerExchange, parity: int, shard: TileShard, N: int, C: int, weights: torch.Tensor,
                              dtype: torch.dtype, out: Optional[torch.Tensor] = None, x_buffer: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Wait for every rank's step counter, then blend reading the peers' chunks over NVLink (one kernel).  With `x_buffer`
    the un-normalised accumulator is stored there as well (region prompt control)."""
    dev = exchange.device
    nb = shard.num_chunks
    ptrs = (ctypes.c_void_p * nb)(*exchange.buf_ptrs[parity][:nb])
    x_out = out if out is not None else torch.empty((N, C, g.H, g.W), dtype=torch.float32, device=dev)
    if g.wrap:   # a periodic plan: the windowed wrap blend over the whole canvas, waiting for every rank, no own bands
        wait = (ctypes.c_void_p(exchange.flag_ptrs[exchange.rank]), exchange.world, ctypes.c_void_p(exchange.counter_ptr))
        return engine.blend_multidiffusion_wrap_rows(g, list(exchange.buf_ptrs[parity][:nb]), N, C, dtype, weights, x_out, 0, g.H,
                                                     x_buffer=x_buffer, wait=wait, tile_bs=shard.chunk)
    with torch.cuda.device(dev):
        check(lib.td_blend_multidiffusion_peer(ctypes.byref(g), ptrs, nb, shard.chunk, N, C, _cabi.dtype_code(dtype),
                                               _cabi.dtype_code(dtype), weights.data_ptr(), x_out.data_ptr(),
                                               x_buffer.data_ptr() if x_buffer is not None else None,
                                               ctypes.c_void_p(exchange.flag_ptrs[exchange.rank]), exchange.world,
                                               ctypes.c_void_p(exchange.counter_ptr), 0, _cabi.current_stream_ptr(dev)))
    return x_out


# ===================================================================================================================
# Row-strip tile shard with halo-only exchange (the default multi-GPU form of MultiDiffusion)
# ===================================================================================================================
class StripShard:
    """Row-strip partition of a grid plan over `world` ranks (pure bookkeeping, no device work).

    Rank r denoises the tiles of a contiguous run of tile ROWS ("bands") and owns the canvas rows
    `[B[r], B[r+1])`, B[r] = the first band's origin rounded down to a multiple of 8 (B[0] = 0, B[world] = H).  A canvas
    row is covered by the bands whose extent `[ys[i], ys[i] + th)` contains it; for a row of rank r these are its own
    bands and bands of LOWER ranks that reach down into the strip (never higher ones: they start at or below
    B[r+1]).  So per sampler step
      * tile halo, down the ranks: rank p sends rank q > p the rows `[v0, v1)` of every tile of band i that fall
        into q's strip (`halo_out` / `halo_in`) -- at BASELINE cfg2 about 54 tile rows per boundary instead of the
        whole tile list;
      * latent halo, up the ranks: rank r scatters from canvas rows `[ys[first band], ys[last band] + th)`, which
        reach into the strips of higher ranks; they send those rows of the blended latent back (`x_out` / `x_in`).
    Every pixel is blended by exactly one rank, with the covering tiles in the same ascending order as on one GPU:
    the union of the strips is bit-identical to the single-GPU latent.

    `wrap_y` (a plan periodic in y, seamless tiling): band i covers the canvas rows (ys[i] + v) mod H, v < tile_h, so the
    last band(s) run past H into the top rows of rank 0's strip (on a pitch-4 plan also of further strips) -- the strips
    close into a ring.  Tile halo then also goes "down" across the seam (rank W-1 -> rank 0), a rank whose bands wrap
    scatters from the rows [ys[first], H) and [0, e) and receives the top ones from their owners, and a waiter's senders
    may be a cyclic run of ranks, e.g. {W-1, 0} (see the flag bookkeeping below).  Rows keep their canvas position."""

    def __init__(self, ys: Sequence[int], cols: int, tile_h: int, H: int, rank: int, world: int, wrap_y: bool = False):
        if not (0 <= rank < world):
            raise ValueError(f"rank {rank} outside world {world}")
        rows = len(ys)
        self.rank, self.world, self.rows, self.cols, self.tile_h, self.H = rank, world, rows, cols, tile_h, H
        self.wrap_y = bool(wrap_y)
        self.ys = [int(v) for v in ys]
        base, extra = divmod(rows, world)
        counts = [base + (1 if r < extra else 0) for r in range(world)]
        self.band_begin = [sum(counts[:r]) for r in range(world)]
        self.band_end = [self.band_begin[r] + counts[r] for r in range(world)]
        B = []
        for r in range(world):
            if counts[r] == 0:
                B.append(H)
            else:
                B.append(0 if self.band_begin[r] == 0 else self.ys[self.band_begin[r]] // 8 * 8)
        B.append(H)
        for r in range(world - 1, -1, -1):      # monotone (overlap > tile pitch could put a later origin first)
            B[r] = min(B[r], B[r + 1])
        self.B = B

    # ---- per-rank views ---------------------------------------------------------------------------------------
    def bands(self, r: Optional[int] = None) -> range:
        r = self.rank if r is None else r
        return range(self.band_begin[r], self.band_end[r])

    def tile_range(self, r: Optional[int] = None):
        r = self.rank if r is None else r
        return self.band_begin[r] * self.cols, self.band_end[r] * self.cols

    def strip(self, r: Optional[int] = None):
        r = self.rank if r is None else r
        return self.B[r], self.B[r + 1]

    def owner_of_band(self, i: int) -> int:
        for r in range(self.world):
            if self.band_begin[r] <= i < self.band_end[r]:
                return r
        raise IndexError(i)

    def halo_in(self, r: Optional[int] = None):
        """[(band i, owner rank, v0, v1)]: tile rows [v0, v1) of every tile of band i (not r's own) that rank r blends."""
        r = self.rank if r is None else r
        lo, hi = self.strip(r)
        out = []
        if hi <= lo:
            return out
        for i in range(self.rows):
            if self.band_begin[r] <= i < self.band_end[r]:
                continue
            v0, v1 = max(0, lo - self.ys[i]), min(self.tile_h, hi - self.ys[i])
            if self.wrap_y:           # the band's rows past H, at v = row - ys[i] + H
                w0, w1 = max(0, lo - self.ys[i] + self.H), min(self.tile_h, hi - self.ys[i] + self.H)
                if w1 > w0:
                    # one contiguous run of tile rows per (band, target): the pushes and the halo slots rely on it
                    assert v1 <= v0 or v1 == w0, f"band {i} reaches rank {r}'s strip in two separate runs of tile rows"
                    v0, v1 = (v0, w1) if v1 > v0 else (w0, w1)
            if v1 > v0:
                out.append((i, self.owner_of_band(i), v0, v1))
        return out

    def halo_out(self, r: Optional[int] = None):
        """[(band i, destination rank, v0, v1)] of rank r's own bands."""
        r = self.rank if r is None else r
        return [(i, q, v0, v1) for q in range(self.world) if q != r for (i, p, v0, v1) in self.halo_in(q) if p == r]

    def scatter_rows(self, r: Optional[int] = None):
        """Canvas rows rank r reads when it scatters its tiles (under wrap_y the end may lie past H: rows mod H)."""
        r = self.rank if r is None else r
        if self.band_end[r] == self.band_begin[r]:
            return 0, 0
        return self.ys[self.band_begin[r]], self.ys[self.band_end[r] - 1] + self.tile_h

    def scatter_spans(self, r: Optional[int] = None) -> List[tuple]:
        """scatter_rows as canvas row ranges [a, b) inside [0, H): one, or under wrap_y two ([ys_first, H) and [0, e))."""
        lo, hi = self.scatter_rows(r)
        if hi <= self.H:
            return [(lo, hi)] if hi > lo else []
        if hi - self.H >= lo:
            return [(0, self.H)]
        return [(0, hi - self.H), (lo, self.H)]

    def x_in(self, r: Optional[int] = None):
        """[(owner rank q, y0, y1)]: blended-latent rows outside r's strip that r needs for its next scatter."""
        r = self.rank if r is None else r
        spans = self.scatter_spans(r)
        out = []
        for q in range(self.world):
            if q == r:
                continue
            for lo, hi in spans:
                a, b = max(lo, self.B[q]), min(hi, self.B[q + 1])
                if b > a:
                    out.append((q, a, b))
        return out

    def x_out(self, r: Optional[int] = None):
        r = self.rank if r is None else r
        return [(p, a, b) for p in range(self.world) if p != r for (q, a, b) in self.x_in(p) if q == r]

    # ---- flag bookkeeping of the two pushes of a step ("tiles": tile halo, "x": latent halo) ------------------------
    # A waiter polls ONE contiguous run of flag slots, the span of the ranks that send it rows.  The span may hold a rank
    # that has no rows for it (the latent-halo senders of a pitch-4 plan can skip a rank whose strip is empty), and such a
    # rank must still bump its slot every step or the wait never ends: every rank inside a waiter's span pushes to it once
    # per step, a signal-only push (no regions) when it has nothing to send.
    #
    # On a ring (wrap_y) a waiter's senders may be a CYCLIC run, e.g. {W-1, 0}: the span is then the shortest cyclic run from
    # the first sender above the waiter to the last one below it (it never holds the waiter), and it is polled as the
    # contiguous slots [first, first + count) with first + count up to 2 * world: flag slot r + world stands for rank r.  A sender
    # whose rank lies in the wrapped part of a target's run publishes into its mirrored slot r + world there instead of slot r,
    # so td_push_regions and the in-kernel waits stay those of a bounded plan (the flag arrays hold 32 slots, 2 * TD_MAX_PEERS)
    # and a push still publishes into one slot per target (at most world - 1).
    #
    # No wait cycle can stall a step: every wait of step s is satisfied by pushes of step s only, and those pushes are ordered
    # after nothing but the waits of step s - 1 (tile-halo push -> blend -> latent-halo push + wait on each rank).  Nor can a
    # halo be overwritten while it is read: a rank that sends tile halo to q reads latent rows of q (its band covers rows of
    # q's strip, so it scatters from them) and therefore waits, at the end of step s, for q's latent push -- which q makes
    # only after its step-s blend has read that halo.  (Bounded plans: the tile-halo span runs over lower ranks, the
    # latent-halo span over higher ones.)
    def _flag_plan(self):
        if not hasattr(self, "_flag_plan_cache"):
            plan = {}
            W = self.world
            for kind in ("tiles", "x"):
                spans = []
                for r in range(W):
                    s = sorted({p for (_, p, _, _) in self.halo_in(r)}) if kind == "tiles" else sorted({q for (q, _, _) in self.x_in(r)})
                    if not s:
                        spans.append((0, 0))
                    elif not self.wrap_y:
                        spans.append((s[0], s[-1] - s[0] + 1))
                    else:
                        first = next((r + k) % W for k in range(1, W) if (r + k) % W in s)
                        last = next((r - k) % W for k in range(1, W) if (r - k) % W in s)
                        spans.append((first, (last - first) % W + 1))
                holds = lambda q, k: spans[q][0] <= k < spans[q][0] + spans[q][1]
                targets = [[q for q in range(W) if holds(q, r) or holds(q, r + W)] for r in range(W)]
                mirrored = [[q for q in targets[r] if not holds(q, r)] for r in range(W)]
                plan[kind] = (spans, targets, mirrored)
            self._flag_plan_cache = plan
        return self._flag_plan_cache

    def wait_range(self, kind: str, r: Optional[int] = None):
        """(first, count): rank r's wait of flag set `kind` polls the slots of ranks [first, first + count) (count 0: no wait)."""
        r = self.rank if r is None else r
        return self._flag_plan()[kind][0][r]

    def signallers(self, kind: str, r: Optional[int] = None) -> List[int]:
        """The ranks that must push to rank r in set `kind` every step: exactly those of its wait range."""
        first, count = self.wait_range(kind, r)
        return list(range(first, first + count))

    def push_targets(self, kind: str, r: Optional[int] = None) -> List[int]:
        """The ranks rank r pushes to in set `kind` every step (with rows, or signal-only), ascending."""
        r = self.rank if r is None else r
        return list(self._flag_plan()[kind][1][r])

    def mirrored_targets(self, kind: str, r: Optional[int] = None) -> List[int]:
        """The push targets that poll rank r in the wrapped part of their wait run in set `kind`: rank r publishes into its
        mirrored slot r + world there instead of slot r (none under a bounded plan)."""
        r = self.rank if r is None else r
        return list(self._flag_plan()[kind][2][r])

    def push_slots(self, kind: str, r: Optional[int] = None) -> List[tuple]:
        """[(target rank, flag slot)] rank r bumps in set `kind` every step, one per target, ascending by target."""
        r = self.rank if r is None else r
        mirrored = set(self.mirrored_targets(kind, r))
        return [(q, r + self.world if q in mirrored else r) for q in self.push_targets(kind, r)]


# measurement switches (defaults = the shipped path): TD_STRIP_LATE_WAIT=0 -> every blend CTA waits for the halos (no own-band
# test, no reordered schedule)
_LATE_WAIT = os.environ.get("TD_STRIP_LATE_WAIT", "1") != "0"
# TD_STRIP_OVERLAP_PUSH=1 -> the tile-halo push rides a side stream (the step is bound by the NVLink round trip of the push
# itself, which the receiving blend has to wait for either way, so the caller's stream is the default)
_OVERLAP_PUSH = os.environ.get("TD_STRIP_OVERLAP_PUSH", "0") == "1"


class _PeerFlags:
    """One flag array (slot r = what rank r has published to me) + this rank's device-side expect counter, mapped into
    every rank through CUDA IPC.  A push advances the sender's slot on each target by TD_PUSH_CTAS; a waiter compares
    the slots of its senders with its own expect counter (td_push_regions / td_blend_multidiffusion_rows)."""

    def __init__(self, device, group):
        self.device, self.group = device, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        with torch.cuda.device(device):
            self._buf = _RawCudaBuffer(256)
        self._opened: List[int] = []

    def handle(self) -> bytes:
        return self._buf.handle()

    def open(self, handles: Sequence[bytes]):
        self.ptrs = [0] * self.world
        for r, h in enumerate(handles):
            if r == self.rank:
                self.ptrs[r] = self._buf.ptr
                continue
            p = ctypes.c_void_p()
            check(lib.td_ipc_open(ctypes.create_string_buffer(h, len(h)), ctypes.byref(p)))
            self.ptrs[r] = p.value
            self._opened.append(p.value)

    @property
    def counter_ptr(self) -> int:
        return self._buf.ptr + 128

    def set_expect(self, value: int):
        """Initial value of this set's expect counter (sets whose waiters are advanced through another push's bump_next)."""
        t = self._buf.tensor(self.device)
        t[128:132].view(torch.int32).fill_(int(value))
        torch.cuda.synchronize(self.device)

    def push(self, regions: Sequence[tuple], targets: Sequence[int], wait_first: int = 0, wait_count: int = 0, bump_own: bool = True,
             bump_next: Optional[int] = None, mirrored: Sequence[int] = ()):
        """Copy `regions` [(src, dst, planes, rows, row_bytes, src_plane_bytes, src_pitch_bytes, dst_plane_bytes,
        dst_pitch_bytes)] (16-byte aligned) into peer memory and publish them in slot `rank` of the `targets`' flag arrays;
        optionally advance this set's expect counter and wait for ranks [wait_first, wait_first + wait_count); optionally
        advance another set's expect counter (device pointer) when done -- ONE launch (td_push_regions).  `mirrored`: the
        targets that poll this rank in its mirrored slot rank + world (a wrapped strip plan, StripShard.mirrored_targets)."""
        regions = list(regions)
        if len(regions) > _cabi.TD_MAX_PUSH_REGIONS:
            raise ValueError(f"{len(regions)} halo regions in one push (TD_MAX_PUSH_REGIONS = {_cabi.TD_MAX_PUSH_REGIONS})")
        slots = [self.ptrs[q] + 4 * (self.rank + (self.world if q in mirrored else 0)) for q in targets if q != self.rank]
        table = (ctypes.c_void_p * max(1, len(slots)))(*slots)
        arr = (_cabi.TdPushRegion * max(1, len(regions)))()
        for k, (src, dst, planes, rows, rb, sp, spi, dp, dpi) in enumerate(regions):
            arr[k] = _cabi.TdPushRegion(src, dst, planes, rows, rb, sp, spi, dp, dpi)
        with torch.cuda.device(self.device):
            check(lib.td_push_regions(arr, len(regions), table, len(slots), ctypes.c_void_p(self.counter_ptr) if (bump_own or wait_count) else None,
                                      ctypes.c_void_p(self.ptrs[self.rank] + 4 * wait_first) if wait_count else None, wait_count,
                                      ctypes.c_void_p(bump_next) if bump_next else None, _cabi.current_stream_ptr(self.device)))

    def wait_args(self, first: int, count: int):
        """(flags pointer, count, value pointer) for a wait on ranks [first, first + count)."""
        return ctypes.c_void_p(self.ptrs[self.rank] + 4 * first), count, ctypes.c_void_p(self.counter_ptr)

    def close(self):
        for p in self._opened:
            lib.td_ipc_close(ctypes.c_void_p(p))
        self._opened = []
        self._buf.free()


class StripExchange:
    """Device side of the row-strip shard: the halo buffer and the blended latent of every rank are cudaMalloc'd
    and mapped into their neighbours through CUDA IPC; halos are PUSHED over NVLink and published in the same launch
    (td_push_regions: 128-bit stores into peer memory, one release add per CTA into the target's flag slot), and awaited
    inside the blend kernel (only by the CTAs that read a halo band) / by the latent-halo push that closes the step.
    No NCCL call on the data path; every launch is replayable from a CUDA graph (all counters live on the device).

    `dtype` is the tile dtype, `latent_dtype` the dtype of the blended latent `x_out`: fp32 for MultiDiffusion (`blend`), the
    latent dtype for Mixture of Diffusers (`blend_mixture`), fp32 again when FOREGROUND regions are composited over it."""

    def __init__(self, shard: StripShard, N: int, C: int, tile_w: int, W: int, dtype: torch.dtype, device: torch.device, group=None,
                 latent_dtype: torch.dtype = torch.float32):
        self.shard, self.N, self.C, self.tw, self.W, self.dtype, self.device, self.group = shard, N, C, tile_w, W, dtype, device, group
        sh = shard
        self.es = torch.empty((), dtype=dtype).element_size()
        self.latent_dtype = latent_dtype
        self.xes = torch.empty((), dtype=latent_dtype).element_size()
        if (W * self.xes) % 16 != 0:      # the latent-halo rows are pushed as 16-byte vectors
            raise ValueError(f"row-strip shard: a {latent_dtype} latent needs W % {16 // self.xes} == 0 (W = {W})")
        for kind in ("tiles", "x"):       # one td_push_regions publishes into at most TD_MAX_PEERS flag slots
            n = len(sh.push_slots(kind))
            if n > _cabi.TD_MAX_PEERS:
                raise ValueError(f"row-strip shard: rank {sh.rank} would publish into {n} {kind} flag slots per push "
                                 f"(TD_MAX_PEERS = {_cabi.TD_MAX_PEERS})")
        self.band_elems = sh.cols * N * C * sh.tile_h * tile_w                 # one band of tiles [cols*N, C, th, tw]
        self.halo_bands = [i for (i, _, _, _) in sh.halo_in()]
        n_own = len(sh.bands())
        with torch.cuda.device(device):
            self._own = torch.empty(max(1, n_own) * self.band_elems, dtype=dtype, device=device)
            self._halo = _RawCudaBuffer(max(1, len(self.halo_bands)) * self.band_elems * self.es)
            self._xout = _RawCudaBuffer(N * C * sh.H * W * self.xes)
            self.flags_tiles, self.flags_x = _PeerFlags(device, group), _PeerFlags(device, group)
            torch.cuda.synchronize(device)
        mine = [self._halo.handle(), self._xout.handle(), self.flags_tiles.handle(), self.flags_x.handle(), self.halo_bands]
        everyone: List[Optional[list]] = [None] * sh.world
        dist.all_gather_object(everyone, mine, group=group)
        self._opened: List[int] = []
        self.peer_halo, self.peer_xout, self.peer_halo_bands = [0] * sh.world, [0] * sh.world, [None] * sh.world
        for r in range(sh.world):
            self.peer_halo_bands[r] = everyone[r][4]
            if r == sh.rank:
                self.peer_halo[r], self.peer_xout[r] = self._halo.ptr, self._xout.ptr
                continue
            for slot, h in ((self.peer_halo, everyone[r][0]), (self.peer_xout, everyone[r][1])):
                p = ctypes.c_void_p()
                check(lib.td_ipc_open(ctypes.create_string_buffer(h, len(h)), ctypes.byref(p)))
                slot[r] = p.value
                self._opened.append(p.value)
        self.flags_tiles.open([e[2] for e in everyone])
        self.flags_x.open([e[3] for e in everyone])
        self.x_out = self._xout.tensor(device).view(latent_dtype).view(N, C, sh.H, W)
        self._side, self._join = None, None
        self.flags_tiles.set_expect(_cabi.TD_PUSH_CTAS)      # the first step's blend waits for ONE push of each sender
        self._tile_wait, self._x_wait = sh.wait_range("tiles"), sh.wait_range("x")
        self._tile_targets, self._x_targets = sh.push_targets("tiles"), sh.push_targets("x")
        self._tile_mirrored, self._x_mirrored = sh.mirrored_targets("tiles"), sh.mirrored_targets("x")
        dist.barrier(group=group)

    # ---- this rank's tile outputs -----------------------------------------------------------------------------
    def own_tiles(self) -> torch.Tensor:
        """[(own bands * cols) * N, C, th, tw]: where the UNet's outputs of this rank's tiles go (tile-major)."""
        sh = self.shard
        n = len(sh.bands()) * sh.cols * self.N
        return self._own[:n * self.C * sh.tile_h * self.tw].view(n, self.C, sh.tile_h, self.tw)

    def push_tile_halos(self):
        """Rows [v0, v1) of every tile of my band i -> the halo slot of band i on rank q (peer memory), then signal:
        one launch (td_push_regions)."""
        sh = self.shard
        plane = sh.tile_h * self.tw * self.es
        planes = sh.cols * self.N * self.C
        regions = []
        for (i, q, v0, v1) in sh.halo_out():
            src = self._own.data_ptr() + ((i - sh.band_begin[sh.rank]) * self.band_elems + v0 * self.tw) * self.es
            slot = self.peer_halo_bands[q].index(i)
            dst = self.peer_halo[q] + (slot * self.band_elems + v0 * self.tw) * self.es
            # rows v0..v1 of a tile are contiguous: one "row" of (v1 - v0) * tw elements per tile plane
            regions.append((src, dst, planes, 1, (v1 - v0) * self.tw * self.es, plane, plane, plane, plane))
        if not self._aligned(regions):
            raise ValueError("row-strip shard: tile width and halo offsets must be multiples of 16 bytes")
        # the blend's expect counter of this set is advanced by the latent-halo push that closed the PREVIOUS step (bump_next):
        # nothing this launch writes is read by this rank's own blend, so it may ride a side stream
        if not _OVERLAP_PUSH:
            self.flags_tiles.push(regions, self._tile_targets, bump_own=False, mirrored=self._tile_mirrored)
            return
        # side stream: this rank's blend waits (in-kernel, only in the CTAs that read a halo) for the NEIGHBOUR's push, not
        # for this one -- the NVLink copy overlaps the blend of the interior rows; push_x_halos_and_wait joins the side
        # stream before the step ends (the tile buffer is rewritten by the next step's denoiser)
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        fork = torch.cuda.Event()
        fork.record(main)
        self._side.wait_event(fork)
        with torch.cuda.stream(self._side):
            self.flags_tiles.push(regions, self._tile_targets, bump_own=False, mirrored=self._tile_mirrored)
            self._join = torch.cuda.Event()
            self._join.record(self._side)

    @staticmethod
    def _aligned(regions) -> bool:
        return all(v % 16 == 0 for r in regions for v in (r[0], r[1], r[4], r[5], r[6], r[7], r[8]))

    def band_pointer_table(self):
        """One pointer per tile row for td_blend_multidiffusion_rows: own band, halo slot, or (unused) my buffer."""
        sh = self.shard
        ptrs = []
        for i in range(sh.rows):
            if sh.band_begin[sh.rank] <= i < sh.band_end[sh.rank]:
                ptrs.append(self._own.data_ptr() + (i - sh.band_begin[sh.rank]) * self.band_elems * self.es)
            elif i in self.halo_bands:
                ptrs.append(self._halo.ptr + self.halo_bands.index(i) * self.band_elems * self.es)
            else:
                ptrs.append(self._own.data_ptr())
        return (ctypes.c_void_p * sh.rows)(*ptrs)

    def blend(self, g, weights: torch.Tensor, rcp_weights: Optional[torch.Tensor], flags: int = 0,
              x_buffer: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Blend this rank's strip into its IPC-mapped latent buffer (waits in-kernel for the tile halos).  With `x_buffer`
        ([N, C, H, W] of the latent dtype) the un-normalised accumulator of the strip's rows is stored there as well (the
        region composite starts from it)."""
        sh = self.shard
        lo, hi = sh.strip()
        f, count, v = self.flags_tiles.wait_args(*self._tile_wait)
        if hi <= lo:                       # this rank owns no canvas rows (more ranks than tile rows)
            return self.x_out
        if not hasattr(self, "_ptr_table"):
            self._ptr_table = self.band_pointer_table()
        own = (sh.band_begin[sh.rank], sh.band_end[sh.rank]) if _LATE_WAIT else (0, 0)
        if g.wrap:                         # a periodic plan: the windowed wrap blend (no reciprocal weights)
            engine.blend_multidiffusion_wrap_rows(g, list(self._ptr_table), self.N, self.C, self.dtype, weights, self.x_out, lo, hi,
                                                  x_buffer=x_buffer, wait=(f, count, v), own_bands=own, flags=flags)
            return self.x_out
        with torch.cuda.device(self.device):
            check(lib.td_blend_multidiffusion_rows(ctypes.byref(g), self._ptr_table, sh.rows, sh.cols, self.N, self.C, _cabi.dtype_code(self.dtype),
                                                   _cabi.dtype_code(self.dtype), weights.data_ptr(),
                                                   rcp_weights.data_ptr() if rcp_weights is not None else None, self.x_out.data_ptr(),
                                                   x_buffer.data_ptr() if x_buffer is not None else None, lo, hi, f if count else None, count, v if count else None,
                                                   sh.band_begin[sh.rank] if _LATE_WAIT else 0, sh.band_end[sh.rank] if _LATE_WAIT else 0, int(flags),
                                                   _cabi.current_stream_ptr(self.device)))
        return self.x_out

    def blend_mixture(self, g, tile_weights: torch.Tensor, rescale: torch.Tensor, flags: int = 0,
                      x_buffer: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Mixture of Diffusers: the gaussian blend of this rank's strip (waits in-kernel for the tile halos) into its
        IPC-mapped latent buffer, or into `x_buffer` ([N, C, H, W] of the latent dtype) instead when regions are composited
        over the strip next.  Returns the buffer written."""
        from . import engine
        sh = self.shard
        lo, hi = sh.strip()
        out = x_buffer if x_buffer is not None else self.x_out
        if hi <= lo:                       # this rank owns no canvas rows (more ranks than tile rows)
            return out
        if not hasattr(self, "_ptr_table"):
            self._ptr_table = self.band_pointer_table()
        own = (sh.band_begin[sh.rank], sh.band_end[sh.rank]) if _LATE_WAIT else (0, 0)
        rows_blend = engine.blend_mixture_wrap_rows if g.wrap else engine.blend_mixture_rows
        return rows_blend(g, list(self._ptr_table), self.N, self.C, self.dtype, tile_weights, rescale, out, lo, hi,
                          wait=self.flags_tiles.wait_args(*self._tile_wait), own_bands=own, flags=flags)

    def join_side(self):
        """The caller's stream waits for the side-stream tile-halo push of this step (no-op when there is none)."""
        if self._join is not None:
            torch.cuda.current_stream(self.device).wait_event(self._join)
            self._join = None

    def push_x_halos_and_wait(self):
        """Rows of my strip that lower ranks scatter from -> their latent buffers; then wait for mine to arrive
        (copy + signal + wait in one launch: td_push_regions).  Every rank whose wait range holds mine is signalled, also
        one I send no rows to (StripShard.push_targets)."""
        sh = self.shard
        regions = []
        row = self.W * self.xes
        plane = sh.H * row
        for (p, a, b) in sh.x_out():
            regions.append((self._xout.ptr + a * row, self.peer_xout[p] + a * row, self.N * self.C, 1, (b - a) * row, plane, plane, plane, plane))
        first, count = self._x_wait
        self.join_side()
        self.flags_x.push(regions, self._x_targets, first, count, bump_own=True, bump_next=self.flags_tiles.counter_ptr,
                          mirrored=self._x_mirrored)

    def gather_latent(self, x: torch.Tensor) -> torch.Tensor:
        """All ranks' strips of `x` (any tensor laid out like the latent) -> the full latent on every rank."""
        sh = self.shard
        rows = max(sh.B[r + 1] - sh.B[r] for r in range(sh.world))
        send = torch.zeros((x.shape[0], x.shape[1], rows, x.shape[3]), dtype=x.dtype, device=x.device)
        lo, hi = sh.strip()
        if hi > lo:
            send[:, :, :hi - lo] = x[:, :, lo:hi]
        recv = torch.empty((sh.world,) + tuple(send.shape), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(recv.view(-1), send.view(-1), group=self.group)
        out = torch.empty_like(x)
        for r in range(sh.world):
            a, b = sh.strip(r)
            if b > a:
                out[:, :, a:b] = recv[r][:, :, :b - a]
        return out

    def close(self):
        for p in self._opened:
            lib.td_ipc_close(ctypes.c_void_p(p))
        self._opened = []
        self.flags_tiles.close(); self.flags_x.close()
        self._halo.free(); self._xout.free()
