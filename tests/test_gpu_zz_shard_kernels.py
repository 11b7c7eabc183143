"""The device entries of the multi-GPU tile shard on ONE GPU, with emulated ranks: td_peer_signal / td_peer_wait,
td_push_regions, td_blend_multidiffusion_peer (replicate mode) and td_blend_multidiffusion_rows (row-strip mode), and
three steps of the production parallel.StripExchange with k ranks living in one process.  Every pointer of an emulated
rank is local memory and every flag array is local, so worlds 2-8 run on the real kernels and are compared bit for bit
with the oracle and the reference fixtures.

Safety rule.  No launch that waits (td_peer_wait, td_push_regions with wait_count > 0, the rows blend with wait_count > 0,
the peer blend) is issued before its wait is already satisfied: `_assert_ready` synchronises, reads the flag slots and
the value the launch will compare them with, and asserts every slot has reached it under the kernels' (int32)(v - want)
rule.  A bookkeeping bug therefore becomes a host assertion; no test relies on the bounded spin of the kernels.  "Never
read" is shown with NaN-poisoned buffers, never with invalid pointers.

The file sorts after the other test_gpu_* files for the reason given in test_gpu_late_round1.py.
"""
import ctypes
import threading
import types
from functools import lru_cache

import numpy as np
import pytest
import torch

from helpers import DTYPES, assert_bit_equal, bits, load_golden, sha
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel
from multidiffusion_upscaler_for_automatic1111_b200._cabi import (TD_ERR_INVALID_ARG, TD_ERR_UNSUPPORTED, TD_FLAG_NO_PDL,
                                                                  TD_FLAG_ONE_PLANE, TD_FLAG_PEER_ASYNC, TD_OK, lib)
from oracle import blend, synth, tiling

pytestmark = pytest.mark.gpu

P = _cabi.TD_PUSH_CTAS
MASK = 0xFFFFFFFF


def _i32(v: int) -> int:
    v &= MASK
    return v - (1 << 32) if v >= (1 << 31) else v


def _stream():
    return _cabi.current_stream_ptr()


class _Flags:
    """A flag allocation laid out like production's: uint32 slots at +0, the rank's counter at +128."""

    def __init__(self, slots=0, counter=0):
        self.t = torch.zeros(64, dtype=torch.int32, device="cuda")
        self.t[:32] = _i32(slots)
        self.t[32] = _i32(counter)

    @property
    def ptr(self) -> int:
        return self.t.data_ptr()

    def slot_ptr(self, i: int) -> int:
        return self.ptr + 4 * i

    @property
    def counter_ptr(self) -> int:
        return self.ptr + 128

    def slots(self, n: int = 16):
        torch.cuda.synchronize()
        return [v & MASK for v in self.t[:n].tolist()]

    def counter(self) -> int:
        torch.cuda.synchronize()
        return int(self.t[32].item()) & MASK


def _u32_at(t: torch.Tensor, byte_off: int, n: int):
    return [v & MASK for v in t.view(torch.int32)[byte_off // 4:byte_off // 4 + n].tolist()]


def _assert_ready(slot_values, want: int, what: str, first: int = 0):
    """The safety rule: every slot a launch polls (slots first, first + 1, ...) has reached `want` (int32 wrap-around
    compare, as the kernels)."""
    for k, v in enumerate(slot_values):
        assert _i32(v - want) >= 0, f"{what}: slot {first + k} holds {v}, the launch would wait for {want} -- a push that never comes"


def _ready_flags(flags: _Flags, first: int, count: int, want: int, what: str):
    torch.cuda.synchronize()
    _assert_ready(flags.slots(32)[first:first + count], want, what, first)


def test_safety_helper_catches_an_unsatisfied_slot():
    _assert_ready([5, 7, 0x7FFFFFFF], 5, "ok")
    _assert_ready([3], 0xFFFFFFF0, "ahead across the 2^32 wrap")
    with pytest.raises(AssertionError):
        _assert_ready([5, 4], 5, "one behind")
    with pytest.raises(AssertionError):
        _assert_ready([0xFFFFFFF0], 3, "behind across the wrap")


# ------------------------------------------------------------------------------------------------ 1. signal / wait
def _signal(tables, world, rank, counter_ptr):
    arr = (ctypes.c_void_p * max(1, len(tables)))(*tables)
    return lib.td_peer_signal(arr, world, rank, ctypes.c_void_p(counter_ptr), _stream())


@pytest.mark.parametrize("world", [1, 2, 5, 16])
def test_peer_signal_bumps_the_counter_and_publishes_it(world):
    arrays = [_Flags(slots=0xA5A5A5A5, counter=10 * q) for q in range(world)]
    counters = [10 * q for q in range(world)]
    for rank in sorted({0, world // 2, world - 1}) + [world - 1]:
        old = [a.slots(32) for a in arrays]
        assert _signal([a.ptr for a in arrays], world, rank, arrays[rank].counter_ptr) == TD_OK
        counters[rank] += 1
        assert [a.counter() for a in arrays] == counters, "the signal must bump its own counter by exactly 1, and no other"
        for q, a in enumerate(arrays):
            want = list(old[q])
            want[rank] = counters[rank]
            assert a.slots(32) == want, f"world {world}: array of rank {q} after the signal of rank {rank}"


def test_peer_signal_counter_wraps():
    a = _Flags(counter=MASK)
    assert _signal([a.ptr], 1, 0, a.counter_ptr) == TD_OK
    assert a.counter() == 0 and a.slots(1) == [0]


@pytest.mark.parametrize("value,slots", [(1, [1, 1, 1]), (7, [7, 9, 1000]), (0xFFFFFFF0, [0xFFFFFFF0, 0xFFFFFFFF, 0, 5])])
def test_peer_wait_on_satisfied_flags(value, slots):
    f = _Flags(counter=value)
    for i, v in enumerate(slots):
        f.t[i] = _i32(v)
    _ready_flags(f, 0, len(slots), f.counter(), "td_peer_wait")
    assert lib.td_peer_wait(ctypes.c_void_p(f.ptr), len(slots), ctypes.c_void_p(f.counter_ptr), _stream()) == TD_OK
    torch.cuda.synchronize()
    assert f.slots(len(slots)) == [v & MASK for v in slots]


def test_peer_signal_replayed_from_a_cuda_graph():
    a, b = _Flags(), _Flags()
    table = [a.ptr, b.ptr]
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph, stream=side):
        assert _signal(table, 2, 1, b.counter_ptr) == TD_OK
    assert b.counter() == 0, "capturing ran the signal"
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert b.counter() == 3 and a.slots(2) == [0, 3] and b.slots(2) == [0, 3]


def test_peer_signal_and_wait_argument_statuses():
    a = _Flags()
    tbl = [a.ptr] * 17
    assert _signal(tbl, 0, 0, a.counter_ptr) == TD_ERR_INVALID_ARG
    assert _signal(tbl, 17, 0, a.counter_ptr) == TD_ERR_INVALID_ARG
    assert _signal(tbl, 2, 2, a.counter_ptr) == TD_ERR_INVALID_ARG
    assert _signal(tbl, 2, -1, a.counter_ptr) == TD_ERR_INVALID_ARG
    assert _signal([a.ptr, None, a.ptr], 3, 0, a.counter_ptr) == TD_ERR_INVALID_ARG
    assert lib.td_peer_wait(ctypes.c_void_p(a.ptr), 17, ctypes.c_void_p(a.counter_ptr), _stream()) == TD_ERR_INVALID_ARG
    assert lib.td_peer_wait(None, 1, ctypes.c_void_p(a.counter_ptr), _stream()) == TD_ERR_INVALID_ARG
    assert lib.td_peer_wait(None, 0, None, _stream()) == TD_OK       # nothing to wait for: no launch
    torch.cuda.synchronize()
    assert a.counter() == 0 and a.slots(32) == [0] * 32


# ------------------------------------------------------------------------------------------------ 2. td_push_regions
def _push(regions, target_ptrs, expect_own=None, wait_ptr=None, wait_count=0, bump_next=None):
    arr = (_cabi.TdPushRegion * max(1, len(regions)))()
    for k, r in enumerate(regions):
        arr[k] = _cabi.TdPushRegion(*r)
    tbl = (ctypes.c_void_p * max(1, len(target_ptrs)))(*target_ptrs)
    v = lambda p: ctypes.c_void_p(p) if p else None
    return lib.td_push_regions(arr, len(regions), tbl, len(target_ptrs), v(expect_own), v(wait_ptr), wait_count, v(bump_next), _stream())


def _region_layouts(rng, n):
    """n strided regions (planes, rows, row_bytes, src plane / pitch, dst plane / pitch) from 16 B to several MB."""
    out = []
    for k in range(n):
        big = k % 3 == 2
        planes = int(rng.integers(1, 9)) if big else int(rng.integers(1, 4))
        rows = int(rng.integers(16, 97)) if big else int(rng.integers(1, 6))
        rb = 16 * int(rng.integers(1, 513 if big else 9))
        spi, dpi = rb + 16 * int(rng.integers(0, 5)), rb + 16 * int(rng.integers(0, 5))
        sp, dp = rows * spi + 16 * int(rng.integers(1, 9)), rows * dpi + 16 * int(rng.integers(0, 9))
        if dp == rows * dpi:
            dp += 16 if k % 2 else 0          # some plane strides equal rows * pitch, most do not
        out.append((planes, rows, rb, sp, spi, dp, dpi))
    return out


@pytest.mark.parametrize("n", list(range(1, 9)))
def test_push_regions_copies_exactly_the_regions(n):
    rng = np.random.default_rng(100 + n)
    lay = _region_layouts(rng, n)
    if n == 1:
        lay = [(1, 1, 16, 16, 16, 16, 16)]      # the smallest region: one 16-byte vector
    s_off, d_off, so, do = [], [], 256, 512
    for (planes, rows, rb, sp, spi, dp, dpi) in lay:
        s_off.append(so)
        d_off.append(do)
        so += (planes - 1) * sp + (rows - 1) * spi + rb + 16 * int(rng.integers(1, 4))
        do += (planes - 1) * dp + (rows - 1) * dpi + rb + 16 * int(rng.integers(0, 4))
    src_h = torch.from_numpy(rng.integers(0, 256, size=so + 256, dtype=np.uint8))
    src = src_h.cuda()
    sentinel = 0xA5
    dst = torch.full((do + 512,), sentinel, dtype=torch.uint8, device="cuda")
    want = torch.full((do + 512,), sentinel, dtype=torch.uint8)
    regions = []
    for (planes, rows, rb, sp, spi, dp, dpi), a, b in zip(lay, s_off, d_off):
        regions.append((src.data_ptr() + a, dst.data_ptr() + b, planes, rows, rb, sp, spi, dp, dpi))
        want.as_strided((planes, rows, rb), (dp, dpi, 1), b).copy_(src_h.as_strided((planes, rows, rb), (sp, spi, 1), a))
    total = sum(p * r * rb for (p, r, rb, *_rest) in lay)
    nt = 1 + (n * 5) % 16                      # 1..16 targets
    tgt, own, nxt = _Flags(slots=11), _Flags(counter=1000), _Flags(counter=MASK - 7)
    assert _push(regions, [tgt.slot_ptr(i) for i in range(nt)], expect_own=own.counter_ptr, bump_next=nxt.counter_ptr) == TD_OK
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), want), f"{n} regions ({total} bytes): bytes differ from torch slicing or outside the regions"
    assert tgt.slots(32) == [11 + P] * nt + [11] * (32 - nt)
    assert own.counter() == 1000 + P and nxt.counter() == (MASK - 7 + P) & MASK
    # NULL expect_own / bump_next leave every counter alone
    assert _push(regions, [tgt.slot_ptr(0)]) == TD_OK
    assert tgt.slots(2) == [11 + 2 * P, 11 + P] and tgt.counter() == 0 and own.counter() == 1000 + P
    assert torch.equal(dst.cpu(), want)


@pytest.mark.parametrize("nt", [1, 3, 16])
def test_push_regions_signal_only(nt):
    """No regions: the targets' slots still advance by TD_PUSH_CTAS (the push of a rank with no rows for its waiter)."""
    tgt, own = _Flags(), _Flags(counter=64)
    assert _push([], [tgt.slot_ptr(i) for i in range(nt)], expect_own=own.counter_ptr) == TD_OK
    assert tgt.slots(16) == [P] * nt + [0] * (16 - nt) and own.counter() == 64 + P


@pytest.mark.parametrize("wait_count", [1, 4, 16])
def test_push_regions_waits_on_satisfied_flags(wait_count):
    src = torch.arange(4096, dtype=torch.int32, device="cuda").view(torch.uint8)
    dst = torch.zeros_like(src)
    mine, tgt = _Flags(counter=MASK - 40), _Flags()
    want = (mine.counter() + P) & MASK          # the launch bumps expect_own first, then waits for it
    for i in range(wait_count):
        mine.t[i] = _i32(want + i)              # crosses the 2^32 wrap for some slots
    _ready_flags(mine, 0, wait_count, want, "td_push_regions")
    reg = [(src.data_ptr(), dst.data_ptr(), 4, 8, 512, 4096, 512, 4096, 512)]
    assert _push(reg, [tgt.slot_ptr(3)], expect_own=mine.counter_ptr, wait_ptr=mine.ptr, wait_count=wait_count,
                 bump_next=tgt.counter_ptr) == TD_OK
    torch.cuda.synchronize()
    assert torch.equal(dst, src) and mine.counter() == want and tgt.counter() == P and tgt.slots(4) == [0, 0, 0, P]


def test_push_regions_argument_statuses():
    f = _Flags()
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    ok = (buf.data_ptr(), buf.data_ptr() + 32, 1, 1, 16, 16, 16, 16, 16)
    assert _push([ok] * 9, [f.ptr]) == TD_ERR_INVALID_ARG                            # > TD_MAX_PUSH_REGIONS
    assert _push([(buf.data_ptr() + 8,) + ok[1:]], [f.ptr]) == TD_ERR_INVALID_ARG    # misaligned source
    assert _push([ok[:4] + (24,) + ok[5:]], [f.ptr]) == TD_ERR_INVALID_ARG           # row length not a multiple of 16
    assert _push([ok[:2] + (0,) + ok[3:]], [f.ptr]) == TD_ERR_INVALID_ARG            # empty region
    assert _push([ok], [f.ptr] * 17) == TD_ERR_INVALID_ARG
    assert _push([ok], [f.ptr], wait_ptr=f.ptr, wait_count=1) == TD_ERR_INVALID_ARG   # a wait needs expect_own
    assert _push([ok], [None]) == TD_ERR_INVALID_ARG
    assert f.slots(32) == [0] * 32 and f.counter() == 0


# ------------------------------------------------------------------------------------------------ shared inputs
@lru_cache(maxsize=None)
def _golden():
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = load_golden(here, "blend_small")
    h = dict(np.load(os.path.join(here, "blend_hashes.npz")))
    cases = {str(n): tuple(int(v) for v in c) for n, c in zip(g["names"], g["cases"])}
    idx = list(h["names"]).index("cfg2_ov48")
    cases["cfg2"] = tuple(int(v) for v in h["cases"][idx])
    return g, h, cases


def _seed_name(name):
    return "cfg2_ov48" if name == "cfg2" else name


@lru_cache(maxsize=None)
def _inputs(case, dn, step=0):
    """(grid, plan, x, tile outputs on the device, fp32 oracle step, un-normalised accumulator) of a geometry."""
    N, C, W, H, tw, th, ov, bs = case[1]
    name = case[0]
    seed = synth.case_seed(_seed_name(name), dn) if step == 0 else 1000 + 17 * step + len(name)
    x = synth.latent(seed, (N, C, H, W), DTYPES[dn])
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, False)
    g = engine.make_grid(W, H, tw, th, ov, bs)
    den = lambda t, bb: synth.fake_denoise(t, bb, N)
    want = blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, den)
    acc = torch.zeros_like(x)
    blend.accumulate_md(acc, den(blend.scatter_tiles(x, plan.bboxes), plan.bboxes), plan.bboxes, N)
    tiles = den(blend.scatter_tiles(x, plan.bboxes), plan.bboxes).cuda()
    return g, plan, x, tiles, want, acc


def _case(name):
    return (name, _golden()[2][name])


def _want_fixture(name, dn, want):
    """The fixture / hash of the reference for a named case; also the oracle (same bits)."""
    g, h, _ = _golden()
    if name == "cfg2":
        assert sha(want) == str(h[f"cfg2_ov48_{dn}_md"]), "oracle differs from the reference hash"
    else:
        assert np.array_equal(bits(want), g[f"{name}_{dn}_md"]), "oracle differs from the reference fixture"


# ------------------------------------------------------------------------------------------------ 3. peer blend (replicate mode)
PEER_CASES = ["a", "b", "d", "e", "cfg2"]


@pytest.mark.parametrize("name", PEER_CASES)
@pytest.mark.parametrize("dn", list(DTYPES))
def test_peer_blend_emulated_worlds(name, dn):
    case = _case(name)
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, x, tiles, want, acc = _inputs(case, dn)
    _want_fixture(name, dn, want)
    T = g.num_tiles
    dt = DTYPES[dn]
    weights = torch.from_numpy(plan.weights).cuda()
    want_d, acc_d = want.cuda(), acc.cuda()
    plane = N * C * th * tw
    for world in range(1, 9):
        shards = [parallel.TileShard(T, r, world) for r in range(world)]
        sh0 = shards[0]
        bufs = []
        for sh in shards[:sh0.num_chunks]:
            b = torch.full((sh.chunk * plane,), float("nan"), dtype=dt, device="cuda")      # the last chunk's padding is NaN
            b[:sh.num_local * plane] = tiles[sh.begin * N:sh.end * N].reshape(-1)
            bufs.append(b)
        flags = [_Flags() for _ in range(world)]
        for r in range(world):
            assert _signal([f.ptr for f in flags], world, r, flags[r].counter_ptr) == TD_OK
        for me in sorted({0, world - 1}):
            ex = types.SimpleNamespace(buf_ptrs=[[b.data_ptr() for b in bufs]] * 2, flag_ptrs=[f.ptr for f in flags], rank=me,
                                       world=world, counter_ptr=flags[me].counter_ptr, device=torch.device("cuda"))
            for fl in (0, TD_FLAG_PEER_ASYNC, TD_FLAG_NO_PDL, TD_FLAG_ONE_PLANE, TD_FLAG_PEER_ASYNC | TD_FLAG_NO_PDL):
                for with_buf in (False, True):
                    xb = torch.full_like(x, float("nan")).cuda() if with_buf else None
                    _ready_flags(flags[me], 0, world, flags[me].counter(), "peer blend")
                    out = _peer_blend(g, ex, sh0, N, C, weights, dt, xb, fl)
                    torch.cuda.synchronize()
                    what = f"{name} {dn} world {world} rank {me} flags {fl:#x}"
                    if not _same_bits(out, want_d):
                        assert_bit_equal(out.cpu(), want, what)
                    if with_buf and not _same_bits(xb, acc_d):
                        assert_bit_equal(xb.cpu(), acc, what + " x_buffer")


def _same_bits(a, b):
    iv = torch.int32 if a.element_size() == 4 else torch.int16
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(iv), b.view(iv))


def _peer_blend(g, ex, shard, N, C, weights, dt, x_buffer, flags):
    """parallel.blend_multidiffusion_peer with kernel flags (the production call passes none)."""
    if flags == 0:
        return parallel.blend_multidiffusion_peer(g, ex, 0, shard, N, C, weights, dt, x_buffer=x_buffer)
    nb = shard.num_chunks
    ptrs = (ctypes.c_void_p * nb)(*ex.buf_ptrs[0][:nb])
    out = torch.empty((N, C, g.H, g.W), dtype=torch.float32, device="cuda")
    _cabi.check(lib.td_blend_multidiffusion_peer(ctypes.byref(g), ptrs, nb, shard.chunk, N, C, _cabi.dtype_code(dt), _cabi.dtype_code(dt),
                                                 weights.data_ptr(), out.data_ptr(), x_buffer.data_ptr() if x_buffer is not None else None,
                                                 ctypes.c_void_p(ex.flag_ptrs[ex.rank]), ex.world, ctypes.c_void_p(ex.counter_ptr), flags,
                                                 _stream()))
    return out


def test_peer_blend_refusals():
    case = _case("b")
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, x, tiles, want, acc = _inputs(case, "f16")
    weights = torch.from_numpy(plan.weights).cuda()
    f = _Flags()
    assert _signal([f.ptr], 1, 0, f.counter_ptr) == TD_OK
    ptrs = (ctypes.c_void_p * 1)(tiles.data_ptr())
    out = torch.empty(N * C * H * W + 4, dtype=torch.float32, device="cuda")

    def call(tile_dt, acc_dt, out_ptr, gg=g):
        return lib.td_blend_multidiffusion_peer(ctypes.byref(gg), ptrs, 1, gg.num_tiles, N, C, tile_dt, acc_dt, weights.data_ptr(), out_ptr,
                                                None, ctypes.c_void_p(f.ptr), 1, ctypes.c_void_p(f.counter_ptr), 0, _stream())
    _ready_flags(f, 0, 1, f.counter(), "peer blend")
    assert call(_cabi.TD_F16, _cabi.TD_F32, out.data_ptr()) == TD_ERR_UNSUPPORTED           # mixed dtypes
    assert call(_cabi.TD_F16, _cabi.TD_F16, out.data_ptr() + 4) == TD_ERR_UNSUPPORTED       # misaligned output
    gc = engine.make_grid(57, 43, 16, 16, 12, 8)                                            # 57 wide: no vector path
    assert lib.td_blend_multidiffusion_peer(ctypes.byref(gc), ptrs, 1, gc.num_tiles, 1, 4, _cabi.TD_F16, _cabi.TD_F16, weights.data_ptr(),
                                            out.data_ptr(), None, ctypes.c_void_p(f.ptr), 1, ctypes.c_void_p(f.counter_ptr), 0,
                                            _stream()) == TD_ERR_UNSUPPORTED
    assert lib.td_blend_multidiffusion_peer(ctypes.byref(g), ptrs, 1, g.num_tiles, N, C, _cabi.TD_F16, _cabi.TD_F16, weights.data_ptr(),
                                            out.data_ptr(), None, ctypes.c_void_p(f.ptr), 17, ctypes.c_void_p(f.counter_ptr), 0,
                                            _stream()) == TD_ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------------ 4. rows blend (strip mode)
# N, C, W, H, tile_w, tile_h, overlap, tile_bs
ROW_PLANS = {
    "a": None, "b": None, "d": None, "e": None, "cfg2": None,
    "h61": (2, 4, 64, 61, 16, 16, 8, 4),            # H not a multiple of 8: the last window ends at H
    "p4_16": (1, 4, 16, 28, 16, 16, 12, 4),         # tile pitch 4 (overlap = tile - 4)
    "p4_32": (2, 4, 32, 44, 32, 32, 28, 4),
    "p4_96": (1, 4, 96, 108, 96, 96, 92, 4),
}
NAN_BITS = {torch.float16: 0x7E5A, torch.bfloat16: 0x7FDA, torch.float32: 0x7FC0_5A5A}


def _row_case(name):
    return _case(name) if ROW_PLANS[name] is None else (name, ROW_PLANS[name])


def _sentinel(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    t.view(torch.int32 if dtype == torch.float32 else torch.int16).fill_(NAN_BITS[dtype])
    return t


def _band_table(sh, tiles, cols, N, keep):
    """The production layout of band_pointer_table: own bands hold the real outputs; a halo band is a copy whose rows
    outside [v0, v1) are NaN; bands that do not touch the window point at a NaN-filled band."""
    band = cols * N
    b0, b1 = sh.band_begin[sh.rank], sh.band_end[sh.rank]
    own = tiles[b0 * band:b1 * band].clone()
    nan = torch.full_like(tiles[:band], float("nan"))
    halo = {}
    for (i, _, v0, v1) in sh.halo_in():
        h = tiles[i * band:(i + 1) * band].clone()
        h[:, :, :v0] = float("nan")
        h[:, :, v1:] = float("nan")
        halo[i] = h
    keep += [own, nan] + list(halo.values())
    bb = band * tiles[0].numel() * tiles.element_size()
    ptrs = [own.data_ptr() + (i - b0) * bb if b0 <= i < b1 else (halo[i].data_ptr() if i in halo else nan.data_ptr()) for i in range(sh.rows)]
    return (ctypes.c_void_p * sh.rows)(*ptrs)


def _rows_call(g, table, sh, N, C, dt, weights, rcp, x_out, x_buf, lo, hi, flags_obj, wait, own, kflags, tile_dt=None):
    first, count = wait
    fptr = ctypes.c_void_p(flags_obj.slot_ptr(first)) if count else None
    vptr = ctypes.c_void_p(flags_obj.counter_ptr) if count else None
    return lib.td_blend_multidiffusion_rows(ctypes.byref(g), table, g.rows, g.cols, N, C, _cabi.dtype_code(tile_dt or dt), _cabi.dtype_code(dt),
                                            weights.data_ptr(), rcp.data_ptr() if rcp is not None else None, x_out.data_ptr(),
                                            x_buf.data_ptr() if x_buf is not None else None, lo, hi, fptr, count, vptr, own[0], own[1],
                                            kflags, _stream())


def _wait_modes(sh, g, lo, hi):
    """(name, (first, count), (own_begin, own_end)) of the four wait settings of one rank's window; all give the same bits."""
    first, count = sh.wait_range("tiles")
    prod = (first, count) if count else (0, 1)        # rank 0 has no tile senders: still take the own-band path
    b0, b1 = sh.band_begin[sh.rank], sh.band_end[sh.rank]
    touching = [i for i in range(g.rows) if g.ys[i] < hi and g.ys[i] + g.tile_h > lo]
    last = touching[-1] if touching else 0
    return [("no wait", (0, 0), (0, 0)),                  # sched 0
            ("own bands", prod, (b0, b1)),                # production's choice (sched 2 when the halo enters from above)
            ("every CTA waits", prod, (0, 0)),
            ("wait at the bottom", prod, (0, last))]      # only patch rows that read the last band wait (sched 1)


@pytest.mark.parametrize("name", list(ROW_PLANS))
@pytest.mark.parametrize("dn", list(DTYPES))
def test_rows_blend_emulated_strips(name, dn):
    case = _row_case(name)
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, x, tiles, want, acc = _inputs(case, dn)
    if ROW_PLANS[name] is None:
        _want_fixture(name, dn, want)
    dt = DTYPES[dn]
    weights = torch.from_numpy(plan.weights).cuda()
    rcp_np = engine.exact_reciprocals(plan.weights)
    rcp = torch.from_numpy(rcp_np).cuda() if rcp_np is not None else None
    want_d, acc_d = want.cuda(), acc.cuda()
    ys = list(g.ys[:g.rows])
    flags = _Flags(slots=5 * P, counter=5 * P)
    for world in (2, 3, 5, 8):
        union = _sentinel((N, C, H, W), torch.float32)
        for r in range(world):
            sh = parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world)
            lo, hi = sh.strip()
            if hi <= lo:
                continue
            keep = []
            table = _band_table(sh, tiles, g.cols, N, keep)
            runs = [(m, w_, o_, 0, use_rcp, use_buf) for (m, w_, o_) in _wait_modes(sh, g, lo, hi)
                    for (use_rcp, use_buf) in ((False, False), (True, True))]
            m, w_, o_ = _wait_modes(sh, g, lo, hi)[1]
            runs += [(m, w_, o_, 0, True, False), (m, w_, o_, 0, False, True),
                     (m, w_, o_, TD_FLAG_NO_PDL, True, True), (m, w_, o_, TD_FLAG_ONE_PLANE, False, True)]
            for (mode, wait, own, kfl, use_rcp, use_buf) in runs:
                x_out = _sentinel((N, C, H, W), torch.float32)
                x_buf = _sentinel((N, C, H, W), dt) if use_buf else None
                sent_out, sent_buf = x_out.clone(), (x_buf.clone() if use_buf else None)
                if wait[1]:
                    _ready_flags(flags, wait[0], wait[1], flags.counter(), "rows blend")
                st = _rows_call(g, table, sh, N, C, dt, weights, rcp if use_rcp else None, x_out, x_buf, lo, hi, flags, wait, own, kfl)
                what = f"{name} {dn} world {world} rank {r} rows [{lo},{hi}) {mode} flags {kfl:#x} rcp {use_rcp} buf {use_buf}"
                assert st == TD_OK, what + ": " + lib.td_last_error().decode()
                torch.cuda.synchronize()
                assert torch.equal(x_out[:, :, lo:hi].view(torch.int32), want_d[:, :, lo:hi].view(torch.int32)), what
                assert torch.equal(x_out[:, :, :lo].view(torch.int32), sent_out[:, :, :lo].view(torch.int32)) and \
                    torch.equal(x_out[:, :, hi:].view(torch.int32), sent_out[:, :, hi:].view(torch.int32)), what + ": rows outside the window written"
                if use_buf:
                    iv = torch.int32 if dt == torch.float32 else torch.int16
                    assert torch.equal(x_buf[:, :, lo:hi].view(iv), acc_d[:, :, lo:hi].view(iv)), what + " x_buffer"
                    assert torch.equal(x_buf[:, :, :lo].view(iv), sent_buf[:, :, :lo].view(iv)) and \
                        torch.equal(x_buf[:, :, hi:].view(iv), sent_buf[:, :, hi:].view(iv)), what + ": x_buffer rows outside the window written"
                union[:, :, lo:hi] = x_out[:, :, lo:hi]
            del keep
        assert_bit_equal(union.cpu(), want, f"{name} {dn} world {world}: union of the strips")
    assert flags.slots(32) == [5 * P] * 32 and flags.counter() == 5 * P


def test_rows_blend_refusals():
    case = _case("b")
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, x, tiles, want, acc = _inputs(case, "f16")
    weights = torch.from_numpy(plan.weights).cuda()
    sh = parallel.StripShard(list(g.ys[:g.rows]), g.cols, g.tile_h, g.H, 0, 1)
    keep = []
    table = _band_table(sh, tiles, g.cols, N, keep)
    f = _Flags()
    x_out = _sentinel((N, C, H, W), torch.float32)
    sent = x_out.clone()
    call = lambda lo, hi, own=(0, 0), tile_dt=None, gg=g: _rows_call(gg, table, sh, N, C, torch.float16, weights, None, x_out, None, lo, hi, f,
                                                                     (0, 0), own, 0, tile_dt=tile_dt)
    assert call(4, 16) == TD_ERR_INVALID_ARG                    # window not on a multiple of 8
    assert call(8, 12) == TD_ERR_INVALID_ARG                    # end not on a multiple of 8 and not H
    assert call(16, 8) == TD_ERR_INVALID_ARG                    # inverted
    assert call(0, H + 8) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(0, g.rows + 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(-1, 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(2, 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, tile_dt=torch.float32) == TD_ERR_UNSUPPORTED   # mixed dtypes
    assert call(8, 8) == TD_OK                                  # empty window: nothing launched, nothing written
    gc = engine.make_grid(57, 43, 16, 16, 12, 8)                # case "c", 57 wide: no vector path
    tc = (ctypes.c_void_p * gc.rows)(*([tiles.data_ptr()] * gc.rows))
    wc = torch.ones(43 * 57, dtype=torch.float32, device="cuda")
    xc = torch.empty(4 * 43 * 57, dtype=torch.float32, device="cuda")
    assert lib.td_blend_multidiffusion_rows(ctypes.byref(gc), tc, gc.rows, gc.cols, 1, 4, _cabi.TD_F16, _cabi.TD_F16, wc.data_ptr(), None,
                                            xc.data_ptr(), None, 0, 8, None, 0, None, 0, 0, 0, _stream()) == TD_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert torch.equal(x_out.view(torch.int32), sent.view(torch.int32))


# ------------------------------------------------------------------------------------------------ 5. StripExchange, k ranks in one process
class _ThreadDist:
    """Stand-in for torch.distributed inside parallel: one thread per rank, a barrier for the collectives."""

    def __init__(self, world):
        self.world = world
        self._bar = threading.Barrier(world, timeout=120)
        self._local = threading.local()
        self._slots = [None] * world

    def set_rank(self, r):
        self._local.rank = r

    def get_rank(self, group=None):
        return self._local.rank

    def get_world_size(self, group=None):
        return self.world

    def all_gather_object(self, out, obj, group=None):
        self._slots[self._local.rank] = obj
        self._bar.wait()
        out[:] = list(self._slots)
        self._bar.wait()

    def barrier(self, group=None):
        self._bar.wait()


def _in_process_ipc(monkeypatch):
    """CUDA IPC cannot open a handle in the process that exported it: td_ipc_open looks the handle up among those this
    process took (td_ipc_get_handle still runs), td_ipc_close has nothing to release."""
    real_get = lib.td_ipc_get_handle
    taken = {}

    def get_handle(ptr, out):
        st = real_get(ptr, out)
        if st == TD_OK:
            taken[ctypes.string_at(out, _cabi.TD_IPC_HANDLE_BYTES)] = ptr.value if isinstance(ptr, ctypes.c_void_p) else ptr
        return st

    def ipc_open(handle, ref):
        ref._obj.value = taken[ctypes.string_at(handle, _cabi.TD_IPC_HANDLE_BYTES)]
        return TD_OK
    monkeypatch.setattr(lib, "td_ipc_get_handle", get_handle)
    monkeypatch.setattr(lib, "td_ipc_open", ipc_open)
    monkeypatch.setattr(lib, "td_ipc_close", lambda ptr: TD_OK)


def _build_exchanges(monkeypatch, ys, g, N, C, dt, world):
    fake = _ThreadDist(world)
    monkeypatch.setattr(parallel, "dist", fake)
    _in_process_ipc(monkeypatch)
    shards = [parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world) for r in range(world)]
    exs, errs = [None] * world, []

    def make(r):
        try:
            fake.set_rank(r)
            exs[r] = parallel.StripExchange(shards[r], N, C, g.tile_w, g.W, dt, torch.device("cuda"))
        except BaseException as e:          # reported on the main thread
            errs.append((r, e))
            fake._bar.abort()
    threads = [threading.Thread(target=make, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errs, f"StripExchange construction failed: {errs}"
    torch.cuda.synchronize()
    return shards, exs


def _span(senders):
    """(first, count) of the flag slots a wait polls: the contiguous run from the lowest to the highest rank that sends the
    waiter rows (what the exchange passes to the kernels)."""
    return (min(senders), max(senders) - min(senders) + 1) if senders else (0, 0)


def _raw_u32(buf):
    torch.cuda.synchronize()
    return buf.tensor(torch.device("cuda")).view(torch.int32)


STRIP_RUNS = [("cfg2", "f16", k) for k in (2, 3, 4, 5, 8)] + [("e", "bf16", 3), ("a", "bf16", 5), ("a", "f32", 4), ("d", "f32", 8)] + \
             [("p4_16", "f16", 4), ("p4_32", "f16", 5), ("p4_32", "bf16", 8)]


@pytest.mark.parametrize("name,dn,world", STRIP_RUNS)
def test_strip_exchange_emulated_ranks(monkeypatch, name, dn, world):
    case = _row_case(name)
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, _, _, _, _ = _inputs(case, dn)
    dt = DTYPES[dn]
    ys = list(g.ys[:g.rows])
    torch.cuda.init()
    shards, exs = _build_exchanges(monkeypatch, ys, g, N, C, dt, world)
    try:
        weights = torch.from_numpy(plan.weights).cuda()
        rcp_np = engine.exact_reciprocals(plan.weights) if dt != torch.float32 else None
        rcp = torch.from_numpy(rcp_np).cuda() if rcp_np is not None else None
        bboxes = [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)]
        for ex in exs:
            ex.x_out.view(torch.int32).fill_(NAN_BITS[torch.float32])
        for step in range(1, 4):
            _, _, x, _, want, _ = _inputs(case, dn, step)
            want_d = want.cuda()
            # 1. scatter from the rank's own latent (NaN outside its strip and latent halo), fake denoise, push the tile halos
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                t0, t1 = sh.tile_range()
                if t1 > t0:
                    lat = torch.full((N, C, H, W), float("nan"), dtype=dt, device="cuda")
                    lo, hi = sh.strip()
                    for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]:
                        lat[:, :, a:b] = x[:, :, a:b].cuda()
                    tiles = engine.scatter_tiles(g, lat, tile_begin=t0, tile_end=t1)
                    ex.own_tiles().copy_(synth.fake_denoise(tiles, bboxes[t0:t1], N))
                ex.push_tile_halos()
            # 2. every blend, each after the safety check (tile set: wait on its range for its own expect counter)
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                first, count = _span({p for (_, p, _, _) in sh.halo_in()})
                raw = _raw_u32(ex.flags_tiles._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), _u32_at(raw, 128, 1)[0], f"{name} world {world} step {step}: blend of rank {r}", first)
                ex.blend(g, weights, rcp)
            # 3. latent-halo pushes, highest rank first: every rank a push waits for is higher and has pushed already
            for r in reversed(range(world)):
                sh, ex = shards[r], exs[r]
                first, count = _span({q for (q, _, _) in sh.x_in()})
                raw = _raw_u32(ex.flags_x._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), (_u32_at(raw, 128, 1)[0] + P) & MASK,
                              f"{name} world {world} step {step}: latent-halo push of rank {r}", first)
                ex.push_x_halos_and_wait()
            torch.cuda.synchronize()
            union = torch.full_like(want_d, float("nan"))
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                lo, hi = sh.strip()
                for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]:
                    if b > a:
                        assert torch.equal(ex.x_out[:, :, a:b].view(torch.int32), want_d[:, :, a:b].view(torch.int32)), \
                            f"{name} {dn} world {world} step {step}: rank {r} rows [{a},{b})"
                union[:, :, lo:hi] = ex.x_out[:, :, lo:hi]
                # counters and slots: what the protocol model predicts (TD_PUSH_CTAS per push)
                for senders, fl, expect in (({p for (_, p, _, _) in sh.halo_in()}, ex.flags_tiles, P * (step + 1)),
                                            ({q for (q, _, _) in sh.x_in()}, ex.flags_x, P * step)):
                    raw = _raw_u32(fl._buf)
                    first, count = _span(senders)
                    signal = set(range(first, first + count))
                    assert _u32_at(raw, 0, world) == [P * step if q in signal else 0 for q in range(world)], f"slots of rank {r}, step {step}"
                    assert _u32_at(raw, 128, 1)[0] == expect, f"expect counter of rank {r}, step {step}"
            assert torch.equal(union.view(torch.int32), want_d.view(torch.int32)), f"{name} {dn} world {world} step {step}: union of the strips"
    finally:
        torch.cuda.synchronize()
        for ex in exs:
            ex.close()
