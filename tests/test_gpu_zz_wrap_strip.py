"""Seamless tiling under the row-strip tile shard on ONE GPU: td_blend_multidiffusion_wrap_rows / td_blend_mixture_wrap_rows for
every strip of emulated worlds, their refusals, three steps of the production parallel.StripExchange on wrapped plans with
emulated ranks, and the delegates in strip and fused replicate mode on a one-rank NCCL group (and on several GPUs when the
machine has them) against the unsharded wrapped delegate.

Every result is compared bit for bit (sign of zero included) with the whole-canvas wrap blend on the same plan and with
tests/wrap_oracle.py.  The safety rule of test_gpu_zz_shard_kernels.py holds: no waiting launch is issued before
`_assert_ready` has shown that its flags are satisfied, and "never read" is shown with NaN-poisoned halo bands."""
import ctypes
import os
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel
from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, TD_ERR_UNSUPPORTED, TD_FLAG_NO_PDL, TD_OK, lib
from oracle import synth
from test_gpu_zz_shard_kernels import (NAN_BITS, P, _assert_ready, _band_table, _Flags, _in_process_ipc, _raw_u32, _ready_flags,
                                       _sentinel, _stream, _ThreadDist, _u32_at)

pytestmark = pytest.mark.gpu

XY = wo.WRAP_X | wo.WRAP_Y
# name -> (N, C, W, H, tile_w, tile_h, overlap, wrap)
PLANS = {
    "cfg2 xy": (1, 4, 512, 512, 96, 96, 48, XY),
    "panorama x": (1, 4, 2048, 512, 96, 96, 48, wo.WRAP_X),
    "y": (2, 4, 128, 96, 48, 40, 16, wo.WRAP_Y),
    "x": (2, 4, 64, 48, 24, 16, 8, wo.WRAP_X),
    "pitch 4 xy": (2, 4, 32, 44, 16, 16, 12, XY),
}


def _iv(dt):
    return torch.int32 if dt == torch.float32 else torch.int16


def _same_bits(a, b):
    return a.dtype == b.dtype and torch.equal(a.contiguous().view(_iv(a.dtype)), b.contiguous().view(_iv(b.dtype)))


def _plan_inputs(name, dn, seed=0):
    N, C, W, H, tw, th, ov, wrap = PLANS[name]
    g = engine.make_grid(W, H, tw, th, ov, 4, wrap=wrap)
    plan = wo.WrapPlan(W, H, tw, th, ov, 4, wrap, gaussian=True)
    gen = torch.Generator().manual_seed(seed)
    tiles = (torch.randn((g.num_tiles * N, C, g.tile_h, g.tile_w), generator=gen) * 1.5).to(DTYPES[dn])
    tiles[::7] = -0.0                                    # signed zeros must survive
    return g, plan, tiles


def _shards(g, world):
    ys = list(g.ys[:g.rows])
    return [parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world, wrap_y=bool(g.wrap & wo.WRAP_Y)) for r in range(world)]


def _md_rows(g, table, nb, tile_bs, N, C, dt, weights, x_out, x_buf, lo, hi, flags_obj, wait, own, kflags=0, tile_dt=None):
    first, count = wait
    return lib.td_blend_multidiffusion_wrap_rows(ctypes.byref(g), table, nb, tile_bs, N, C, _cabi.dtype_code(tile_dt or dt), _cabi.dtype_code(dt),
                                                 weights.data_ptr(), x_out.data_ptr(), x_buf.data_ptr() if x_buf is not None else None, lo, hi,
                                                 ctypes.c_void_p(flags_obj.slot_ptr(first)) if count else None, count,
                                                 ctypes.c_void_p(flags_obj.counter_ptr) if count else None, own[0], own[1], kflags, _stream())


def _mod_rows(g, table, nb, tile_bs, N, C, dt, tw_d, rs_d, x_buf, lo, hi, flags_obj, wait, own, kflags=0, tile_dt=None, rs_ptr=None):
    first, count = wait
    return lib.td_blend_mixture_wrap_rows(ctypes.byref(g), table, nb, tile_bs, N, C, _cabi.dtype_code(tile_dt or dt), _cabi.dtype_code(dt),
                                          tw_d.data_ptr(), rs_ptr if rs_ptr is not None else rs_d.data_ptr(), x_buf.data_ptr(), lo, hi,
                                          ctypes.c_void_p(flags_obj.slot_ptr(first)) if count else None, count,
                                          ctypes.c_void_p(flags_obj.counter_ptr) if count else None, own[0], own[1], kflags, _stream())


def _wait_modes(sh, world):
    """(name, (first, count), own bands): none; satisfied, every CTA waits; satisfied with own bands; a run past `world`."""
    first, count = sh.wait_range("tiles")
    prod = (first, count) if count else (0, 1)
    own = (sh.band_begin[sh.rank], sh.band_end[sh.rank])
    return [("no wait", (0, 0), (0, 0)), ("every CTA waits", prod, (0, 0)), ("own bands", prod, own),
            ("run into the mirrored slots", (world - 1, min(world, _cabi.TD_MAX_PEERS)), own)]


# ------------------------------------------------------------------------------------------------ 1. the rows kernels
@pytest.mark.parametrize("name", list(PLANS))
@pytest.mark.parametrize("dn", list(DTYPES))
def test_wrap_rows_blends_emulated_strips(name, dn):
    N, C, W, H = PLANS[name][:4]
    g, plan, tiles = _plan_inputs(name, dn)
    dt = DTYPES[dn]
    outs = [tiles[i * g.tile_bs * N:(i + 1) * g.tile_bs * N] for i in range(g.num_batches)]
    want_md, want_acc = wo.blend_md(outs, plan.batched_bboxes, N, (N, C, H, W), dt, plan.weights)
    want_mod = wo.blend_mod(outs, plan.batched_bboxes, N, (N, C, H, W), dt, plan.tile_weights, plan.rescale_factor)
    weights = torch.from_numpy(plan.weights).cuda()
    tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
    douts = [o.cuda() for o in outs]
    # the whole-canvas wrap blends on the same plan are the yardstick, and they equal the oracle
    whole_buf = torch.empty((N, C, H, W), dtype=dt, device="cuda")
    whole_md = engine.blend_multidiffusion(g, douts, N, C, g.tile_bs, weights, dt, x_buffer=whole_buf)
    whole_mod = engine.blend_mixture(g, douts, N, C, g.tile_bs, tw_d, rs_d, torch.empty((N, C, H, W), dtype=dt, device="cuda"))
    assert _same_bits(whole_md.cpu(), want_md) and _same_bits(whole_buf.cpu(), want_acc) and _same_bits(whole_mod.cpu(), want_mod)
    dtiles = tiles.cuda()
    flags = _Flags(slots=5 * P, counter=5 * P)
    # window [0, H), no wait, the batch table of the whole-canvas call: the whole-canvas bits
    table = (ctypes.c_void_p * g.num_batches)(*[o.data_ptr() for o in douts])
    x_out, x_buf = _sentinel((N, C, H, W), torch.float32), _sentinel((N, C, H, W), dt)
    assert _md_rows(g, table, g.num_batches, g.tile_bs, N, C, dt, weights, x_out, x_buf, 0, H, flags, (0, 0), (0, 0)) == TD_OK
    x_mod = _sentinel((N, C, H, W), dt)
    assert _mod_rows(g, table, g.num_batches, g.tile_bs, N, C, dt, tw_d, rs_d, x_mod, 0, H, flags, (0, 0), (0, 0)) == TD_OK
    torch.cuda.synchronize()
    assert _same_bits(x_out, whole_md) and _same_bits(x_buf, whole_buf) and _same_bits(x_mod, whole_mod), f"{name} {dn}: window [0, H)"
    for world in (2, 3, 5, 8):
        union_md, union_mod = _sentinel((N, C, H, W), torch.float32), _sentinel((N, C, H, W), dt)
        for sh in _shards(g, world):
            lo, hi = sh.strip()
            if hi <= lo:
                continue
            keep = []
            table = _band_table(sh, dtiles, g.cols, N, keep)
            for (mode, wait, own) in _wait_modes(sh, world):
                for kfl in ((0, TD_FLAG_NO_PDL) if mode == "own bands" else (0,)):
                    what = f"{name} {dn} world {world} rank {sh.rank} rows [{lo},{hi}) {mode} flags {kfl:#x}"
                    if wait[1]:
                        _ready_flags(flags, wait[0], wait[1], flags.counter(), what)
                    x_out, x_buf, x_mod = _sentinel((N, C, H, W), torch.float32), _sentinel((N, C, H, W), dt), _sentinel((N, C, H, W), dt)
                    sent_out, sent_buf = x_out.clone(), x_buf.clone()
                    st = _md_rows(g, table, g.rows, g.cols, N, C, dt, weights, x_out, x_buf, lo, hi, flags, wait, own, kfl)
                    assert st == TD_OK, what + ": " + lib.td_last_error().decode()
                    st = _mod_rows(g, table, g.rows, g.cols, N, C, dt, tw_d, rs_d, x_mod, lo, hi, flags, wait, own, kfl)
                    assert st == TD_OK, what + ": " + lib.td_last_error().decode()
                    torch.cuda.synchronize()
                    assert _same_bits(x_out[:, :, lo:hi], whole_md[:, :, lo:hi]), what + " MD"
                    assert _same_bits(x_buf[:, :, lo:hi], whole_buf[:, :, lo:hi]), what + " MD x_buffer"
                    assert _same_bits(x_mod[:, :, lo:hi], whole_mod[:, :, lo:hi]), what + " MoD"
                    for t, s in ((x_out, sent_out), (x_buf, sent_buf), (x_mod, sent_buf)):
                        assert _same_bits(t[:, :, :lo], s[:, :, :lo]) and _same_bits(t[:, :, hi:], s[:, :, hi:]), what + ": rows outside written"
                    union_md[:, :, lo:hi] = x_out[:, :, lo:hi]
                    union_mod[:, :, lo:hi] = x_mod[:, :, lo:hi]
            del keep
        assert_bit_equal(union_md.cpu(), want_md, f"{name} {dn} world {world}: union of the MD strips")
        assert_bit_equal(union_mod.cpu(), want_mod, f"{name} {dn} world {world}: union of the MoD strips")
    assert flags.slots(32) == [5 * P] * 32 and flags.counter() == 5 * P


def test_wrap_rows_refusals():
    N, C, W, H = PLANS["x"][:4]
    g, plan, tiles = _plan_inputs("x", "f16")
    dt = torch.float16
    dtiles = tiles.cuda()
    sh = _shards(g, 1)[0]
    keep = []
    table = _band_table(sh, dtiles, g.cols, N, keep)
    weights = torch.from_numpy(plan.weights).cuda()
    tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
    f = _Flags()
    x_out, x_buf = _sentinel((N, C, H, W), torch.float32), _sentinel((N, C, H, W), dt)
    sent_out, sent_buf = x_out.clone(), x_buf.clone()

    def both(lo, hi, wait=(0, 0), own=(0, 0), tile_dt=None, gg=g, tbl=table):
        a = _md_rows(gg, tbl, gg.rows, gg.cols, N, C, dt, weights, x_out, None, lo, hi, f, wait, own, tile_dt=tile_dt)
        b = _mod_rows(gg, tbl, gg.rows, gg.cols, N, C, dt, tw_d, rs_d, x_buf, lo, hi, f, wait, own, tile_dt=tile_dt)
        assert a == b, (lo, hi, wait, own)
        return a
    bounded = engine.make_grid(W, H, 24, 16, 8, 4)
    assert bounded.rows == g.rows and bounded.cols == g.cols
    assert both(0, 16, gg=bounded) == TD_ERR_UNSUPPORTED         # a bounded plan keeps td_blend_*_rows
    assert both(4, 16) == TD_ERR_INVALID_ARG                     # window not on a multiple of 8
    assert both(8, 12) == TD_ERR_INVALID_ARG                     # end neither on a multiple of 8 nor H
    assert both(16, 8) == TD_ERR_INVALID_ARG                     # inverted
    assert both(0, H + 8) == TD_ERR_INVALID_ARG
    assert both(0, 16, wait=(0, _cabi.TD_MAX_PEERS + 1)) == TD_ERR_INVALID_ARG   # bad wait table
    nul = lib.td_blend_multidiffusion_wrap_rows(ctypes.byref(g), table, g.rows, g.cols, N, C, _cabi.TD_F16, _cabi.TD_F16, weights.data_ptr(),
                                                x_out.data_ptr(), None, 0, 16, ctypes.c_void_p(f.ptr), 2, None, 0, 0, 0, _stream())
    assert nul == TD_ERR_INVALID_ARG                              # a wait without its value pointer
    assert both(0, 16, own=(0, g.rows + 1)) == TD_ERR_INVALID_ARG
    assert both(0, 16, own=(-1, 1)) == TD_ERR_INVALID_ARG
    assert both(0, 16, own=(2, 1)) == TD_ERR_INVALID_ARG
    assert both(0, 16, tile_dt=torch.float32) == TD_ERR_UNSUPPORTED      # mixed dtypes
    assert _mod_rows(g, table, g.rows, g.cols, N, C, dt, tw_d, rs_d, x_buf, 0, 16, f, (0, 0), (0, 0),
                     rs_ptr=rs_d.data_ptr() + 4) == TD_ERR_UNSUPPORTED    # misaligned rescale
    mis = (ctypes.c_void_p * g.rows)(*[table[i] + 2 for i in range(g.rows)])
    assert _md_rows(g, mis, g.rows, g.cols, N, C, dt, weights, x_out, None, 0, 16, f, (0, 0), (0, 0)) == TD_ERR_UNSUPPORTED
    assert both(8, 8) == TD_OK                                   # empty window: nothing launched
    torch.cuda.synchronize()
    assert _same_bits(x_out, sent_out) and _same_bits(x_buf, sent_buf), "a refused call wrote"
    assert f.slots(32) == [0] * 32


# ------------------------------------------------------------------------------------------------ 2. StripExchange, k ranks in one process
def _build_exchanges(monkeypatch, g, N, C, dt, world, latent_dtype):
    fake = _ThreadDist(world)
    monkeypatch.setattr(parallel, "dist", fake)
    _in_process_ipc(monkeypatch)
    import threading
    shards = _shards(g, world)
    exs, errs = [None] * world, []

    def make(r):
        try:
            fake.set_rank(r)
            exs[r] = parallel.StripExchange(shards[r], N, C, g.tile_w, g.W, dt, torch.device("cuda"), latent_dtype=latent_dtype)
        except BaseException as e:
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


def _defer_latent_wait(ex, deferred):
    """On one GPU the latent-halo waits of a ring form a cycle (rank W-1 reads rows of rank 0, rank 0 of rank 1, ...): a push
    that waited in-kernel would block the stream the later pushes need.  The push is issued as in production but without its
    wait; the wait is checked (and then launched, satisfied) after every rank has pushed."""
    real = ex.flags_x.push

    def push(regions, targets, wait_first=0, wait_count=0, bump_own=True, bump_next=None, mirrored=()):
        deferred.append((ex, wait_first, wait_count))
        return real(regions, targets, 0, 0, bump_own=bump_own, bump_next=bump_next, mirrored=mirrored)
    ex.flags_x.push = push


# (plan, dtype, world, method); "pitch 4 xy" at world 4: rank 3's latent halo comes from ranks 0 AND 1
EXCHANGE_RUNS = [("x", "f16", 2, "md"), ("y", "bf16", 3, "mod"), ("pitch 4 xy", "f16", 4, "md"), ("pitch 4 xy", "f32", 4, "mod"),
                 ("pitch 4 xy", "bf16", 8, "md"), ("cfg2 xy", "f16", 5, "mod"), ("cfg2 xy", "f16", 8, "md"), ("y", "f16", 6, "md"),
                 ("x", "bf16", 5, "mod")]


@pytest.mark.parametrize("name,dn,world,method", EXCHANGE_RUNS)
def test_wrap_strip_exchange_emulated_ranks(monkeypatch, name, dn, world, method):
    N, C, W, H = PLANS[name][:4]
    g, plan, _ = _plan_inputs(name, dn)
    dt = DTYPES[dn]
    torch.cuda.init()
    shards, exs = _build_exchanges(monkeypatch, g, N, C, dt, world, torch.float32 if method == "md" else dt)
    if name == "pitch 4 xy" and world == 4:
        assert {q for (q, _, _) in shards[3].x_in()} == {0, 1}
        assert any(sh.mirrored_targets(k) for sh in shards for k in ("tiles", "x"))
    deferred = []
    for ex in exs:
        _defer_latent_wait(ex, deferred)
    try:
        weights = torch.from_numpy(plan.weights).cuda()
        tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
        bboxes = [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)]
        denoise = lambda t, bbs: synth.fake_denoise(t, bbs, N)
        for ex in exs:
            ex.x_out.view(_iv(ex.x_out.dtype)).fill_(NAN_BITS[ex.x_out.dtype])
        for step in range(1, 4):
            x = synth.latent(40 + step, (N, C, H, W), dt)
            want = (wo.multidiffusion_step(x, plan, denoise)[0] if method == "md" else wo.mixture_step(x, plan, denoise)).cuda()
            for sh, ex in zip(shards, exs):
                t0, t1 = sh.tile_range()
                if t1 > t0:
                    lat = torch.full((N, C, H, W), float("nan"), dtype=dt, device="cuda")
                    lo, hi = sh.strip()
                    for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]:
                        lat[:, :, a:b] = x[:, :, a:b].cuda()
                    tiles = engine.scatter_tiles(g, lat, tile_begin=t0, tile_end=t1)
                    ex.own_tiles().copy_(synth.fake_denoise(tiles, bboxes[t0:t1], N))
                ex.push_tile_halos()
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                first, count = sh.wait_range("tiles")
                raw = _raw_u32(ex.flags_tiles._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), _u32_at(raw, 128, 1)[0], f"{name} world {world} step {step}: blend of rank {r}", first)
                if method == "md":
                    ex.blend(g, weights, None)
                else:
                    ex.blend_mixture(g, tw_d, rs_d)
            del deferred[:]
            for ex in exs:
                ex.push_x_halos_and_wait()
            for (ex, first, count) in deferred:
                raw = _raw_u32(ex.flags_x._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), _u32_at(raw, 128, 1)[0], f"{name} world {world} step {step}: latent wait", first)
                if count:
                    assert lib.td_peer_wait(ctypes.c_void_p(ex.flags_x._buf.ptr + 4 * first), count, ctypes.c_void_p(ex.flags_x.counter_ptr),
                                            _stream()) == TD_OK
            torch.cuda.synchronize()
            union = torch.full_like(want, float("nan"))
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                lo, hi = sh.strip()
                for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]:
                    assert _same_bits(ex.x_out[:, :, a:b], want[:, :, a:b]), f"{name} {dn} world {world} step {step}: rank {r} rows [{a},{b})"
                union[:, :, lo:hi] = ex.x_out[:, :, lo:hi]
                for kind, fl, expect in (("tiles", ex.flags_tiles, P * (step + 1)), ("x", ex.flags_x, P * step)):
                    first, count = sh.wait_range(kind)
                    raw = _raw_u32(fl._buf)
                    assert _u32_at(raw, 0, 2 * world) == [P * step if first <= k < first + count else 0 for k in range(2 * world)], \
                        f"{kind} slots of rank {r}, step {step}"
                    assert _u32_at(raw, 128, 1)[0] == expect, f"{kind} expect counter of rank {r}, step {step}"
            assert _same_bits(union, want), f"{name} {dn} world {world} step {step}: union of the strips"
    finally:
        torch.cuda.synchronize()
        for ex in exs:
            ex.close()


# ------------------------------------------------------------------------------------------------ 3. the delegates
GRID = dict(N=2, C=4, W=64, H=48, tw=24, th=16, ov=8, bs=3)
_BG, _FG = "Background", "Foreground"
REGIONS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", _BG, 0.2, -1),
           (True, 0.4, 0.3, 0.45, 0.6, "a dog", "", _FG, 0.3, 5)]


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _delegate(cls, wrap, rows):
    c = GRID
    d = cls(types.SimpleNamespace(width=c["W"] * 8, height=c["H"] * 8, sampler_name="Euler a", disable_extra_networks=True),
            types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None,
                                                                       step=0)))
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"], wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    if rows:
        d.init_custom_bbox({i: row for i, row in enumerate(rows)}, True, False)
    d.init_done()
    return d


def _md_step(d, x):
    return d.sample_one_step(x, None, wo.blur_denoise, lambda xt, i, bb: synth.fake_region_denoise(xt, i)).clone()


def _mod_step(d, x):
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    N = x.shape[0]
    model = types.SimpleNamespace(apply_model=lambda x_tile, t, c_: wo.blur_denoise(x_tile), cond_stage_key="txt",
                                  model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: synth.fake_region_denoise(x_tile, bbox_id)
    d.hook()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4, device=x.device)], "c_concat": [torch.zeros(N, 5, 1, 1, device=x.device)]}
    out = model.apply_model(x, torch.ones(N, device=x.device), cond).clone()
    d.unhook()
    return out


def _gpu_wrap_shard_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    torch.cuda.set_device(rank)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        c = GRID
        N = c["N"]
        host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=None))
        for cls, stepf in ((MultiDiffusion, _md_step), (MixtureOfDiffusers, _mod_step)):
            for wrap in (wo.WRAP_X, XY):
                for rows in ([], REGIONS):
                    xs = [synth.latent(90 + k, (N, c["C"], c["H"], c["W"]), torch.float16) for k in range(3)]
                    wants = [stepf(_delegate(cls, wrap, rows), x.cuda()).cpu() for x in xs]
                    for mode in ("strip", "replicate"):
                        d = _delegate(cls, wrap, rows)
                        with pytest.raises(NotImplementedError, match="explicit"):
                            d.init_tile_shard(None)
                        d.init_tile_shard(None, fused=True, mode=mode)
                        for k, x in enumerate(xs):
                            out = stepf(d, x.cuda())
                            torch.cuda.synchronize()
                            what = f"rank {rank} {cls.__name__} wrap {wrap} regions {len(rows)} {mode} step {k}"
                            assert out.dtype == wants[k].dtype, what
                            if mode == "strip":
                                lo, hi = d._strip.strip()
                                for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in d._strip.x_in()]:
                                    assert _same_bits(out[:, :, a:b].cpu(), wants[k][:, :, a:b]), f"{what}: rows [{a},{b})"
                                dist.barrier()
                                out = d.gather_latent(out)
                            assert _same_bits(out.cpu(), wants[k]), what
                            dist.barrier()
                        dist.barrier()
                        if d._strip_exchange is not None:
                            d._strip_exchange.close()
                        if getattr(d, "_exchange", None) is not None:
                            d._exchange.close()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


def test_one_rank_wrapped_shard_delegates_bit_identical_to_unsharded(tmp_path):
    mp.spawn(_gpu_wrap_shard_worker, args=(1, _free_port(), str(tmp_path)), nprocs=1, join=True)
    assert (tmp_path / "ok0").exists()


def test_multi_gpu_wrapped_shard_delegates_bit_identical_to_one_gpu(tmp_path):
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs 2 GPUs")
    world = min(world, 4)
    mp.spawn(_gpu_wrap_shard_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
