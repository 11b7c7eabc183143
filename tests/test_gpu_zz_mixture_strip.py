"""Mixture of Diffusers under the row-strip tile shard on the GPU: td_blend_mixture_rows for every strip of emulated worlds
against td_blend_mixture and the oracle, its refusals, three steps of the production parallel.StripExchange in its
Mixture-of-Diffusers form with k ranks in one process, and the delegate with init_tile_shard(mode="strip") against the
unsharded delegate (one rank; two or more GPUs when present).

The safety rule of test_gpu_zz_shard_kernels.py holds here: no launch that waits is issued before `_assert_ready` has shown
its flags satisfied, "never read" is shown with NaN-poisoned buffers, and no test relies on the kernels' bounded spin.
The file sorts after the other test_gpu_* files for the reason given in test_gpu_late_round1.py."""
import ctypes
import functools
import os
import types
from functools import lru_cache

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import DTYPES, bits
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel
from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_INVALID_ARG, TD_ERR_UNSUPPORTED, TD_FLAG_NO_PDL, TD_OK, lib
from oracle import blend, synth, tiling
from test_gpu_zz_shard_kernels import (MASK, P, ROW_PLANS, _assert_ready, _band_table, _build_exchanges, _Flags, _golden, _inputs,
                                       _raw_u32, _ready_flags, _row_case, _sentinel, _span, _u32_at, _wait_modes)

pytestmark = pytest.mark.gpu


def _iv(dt):
    return torch.int32 if dt == torch.float32 else torch.int16


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(_iv(a.dtype)), b.contiguous().view(_iv(b.dtype)))


@lru_cache(maxsize=None)
def _mod_inputs(case, dn, step=0):
    """(grid, gaussian plan, tile outputs on the device, oracle latent of the Mixture-of-Diffusers blend) of a geometry; the
    latent and tile outputs are those of test_gpu_zz_shard_kernels._inputs."""
    N, C, W, H, tw, th, ov, bs = case[1]
    g, _, x, tiles, _, _ = _inputs(case, dn, step)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, True)
    want = blend.mixture_step(x, plan.batched_bboxes, plan.tile_weights, plan.rescale_factor, lambda t, bb: synth.fake_denoise(t, bb, N))
    return g, plan, tiles, want


def _mod_rows_call(g, table, N, C, dt, tw_d, rs_d, x_buf, lo, hi, flags_obj, wait, own, kflags, tile_dt=None, tw_ptr=None):
    first, count = wait
    fptr = ctypes.c_void_p(flags_obj.slot_ptr(first)) if count else None
    vptr = ctypes.c_void_p(flags_obj.counter_ptr) if count else None
    return lib.td_blend_mixture_rows(ctypes.byref(g), table, g.rows, g.cols, N, C, _cabi.dtype_code(tile_dt or dt), _cabi.dtype_code(dt),
                                     tw_ptr if tw_ptr is not None else tw_d.data_ptr(), rs_d.data_ptr(), x_buf.data_ptr(), lo, hi, fptr,
                                     count, vptr, own[0], own[1], kflags, _cabi.current_stream_ptr())


# ------------------------------------------------------------------------------------------------ 1. td_blend_mixture_rows
@pytest.mark.parametrize("name", list(ROW_PLANS))
@pytest.mark.parametrize("dn", list(DTYPES))
def test_mixture_rows_blend_emulated_strips(name, dn):
    case = _row_case(name)
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, tiles, want = _mod_inputs(case, dn)
    if ROW_PLANS[name] is None and name != "cfg2":
        assert np.array_equal(bits(want), _golden()[0][f"{name}_{dn}_mod"]), "oracle differs from the reference fixture"
    dt = DTYPES[dn]
    tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
    want_d = want.cuda()
    # the whole-canvas blend (the kernel the windowed launch extends) gives the same bits
    batches = [tiles[b * g.tile_bs * N:min((b + 1) * g.tile_bs, g.num_tiles) * N] for b in range(g.num_batches)]
    whole = engine.blend_mixture(g, batches, N, C, g.tile_bs, tw_d, rs_d, _sentinel((N, C, H, W), dt))
    torch.cuda.synchronize()
    assert _same_bits(whole, want_d), f"{name} {dn}: td_blend_mixture differs from the oracle"
    ys = list(g.ys[:g.rows])
    flags = _Flags(slots=5 * P, counter=5 * P)
    for world in (2, 3, 5, 8):
        union = _sentinel((N, C, H, W), dt)
        for r in range(world):
            sh = parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world)
            lo, hi = sh.strip()
            if hi <= lo:
                continue
            keep = []
            table = _band_table(sh, tiles, g.cols, N, keep)       # halo bands NaN outside the pushed rows
            for (mode, wait, own) in _wait_modes(sh, g, lo, hi):
                for kfl in (0, TD_FLAG_NO_PDL):
                    out = _sentinel((N, C, H, W), dt)
                    sent = out.clone()
                    if wait[1]:
                        _ready_flags(flags, wait[0], wait[1], flags.counter(), "mixture rows blend")
                    st = _mod_rows_call(g, table, N, C, dt, tw_d, rs_d, out, lo, hi, flags, wait, own, kfl)
                    what = f"{name} {dn} world {world} rank {r} rows [{lo},{hi}) {mode} flags {kfl:#x}"
                    assert st == TD_OK, what + ": " + lib.td_last_error().decode()
                    torch.cuda.synchronize()
                    assert _same_bits(out[:, :, lo:hi], want_d[:, :, lo:hi]), what
                    assert _same_bits(out[:, :, :lo], sent[:, :, :lo]) and _same_bits(out[:, :, hi:], sent[:, :, hi:]), \
                        what + ": rows outside the window written"
            union[:, :, lo:hi] = out[:, :, lo:hi]
            del keep
        assert _same_bits(union, want_d), f"{name} {dn} world {world}: union of the strips"
        assert _same_bits(union, whole), f"{name} {dn} world {world}: union differs from td_blend_mixture"
    assert flags.slots(32) == [5 * P] * 32 and flags.counter() == 5 * P


def test_mixture_rows_blend_refusals():
    case = _row_case("b")
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, tiles, want = _mod_inputs(case, "f16")
    tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
    sh = parallel.StripShard(list(g.ys[:g.rows]), g.cols, g.tile_h, g.H, 0, 1)
    keep = []
    table = _band_table(sh, tiles, g.cols, N, keep)
    f = _Flags()
    out = _sentinel((N, C, H, W), torch.float16)
    sent = out.clone()

    def call(lo, hi, own=(0, 0), tile_dt=None, gg=g, tw_ptr=None, tbl=table):
        return _mod_rows_call(gg, tbl, N, C, torch.float16, tw_d, rs_d, out, lo, hi, f, (0, 0), own, 0, tile_dt=tile_dt, tw_ptr=tw_ptr)
    assert call(4, 16) == TD_ERR_INVALID_ARG                    # window not on a multiple of 8
    assert call(8, 12) == TD_ERR_INVALID_ARG                    # end not on a multiple of 8 and not H
    assert call(16, 8) == TD_ERR_INVALID_ARG                    # inverted
    assert call(0, H + 8) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(0, g.rows + 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(-1, 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, own=(2, 1)) == TD_ERR_INVALID_ARG
    assert call(0, 16, tile_dt=torch.float32) == TD_ERR_UNSUPPORTED   # mixed dtypes
    assert call(0, 16, tw_ptr=tw_d.data_ptr() + 4) == TD_ERR_UNSUPPORTED   # tile weights not 16-byte aligned
    assert call(8, 8) == TD_OK                                  # empty window: nothing launched, nothing written
    gc = engine.make_grid(57, 43, 16, 16, 12, 8)                # case "c", 57 wide: no vector path
    tc = (ctypes.c_void_p * gc.rows)(*([tiles.data_ptr()] * gc.rows))
    assert call(0, 8, gg=gc, tbl=tc) == TD_ERR_UNSUPPORTED
    gw = engine.make_grid(W, H, tw, th, ov, bs, wrap=engine.WRAP_X)   # a periodic plan has no row-strip form
    tw_ = (ctypes.c_void_p * gw.rows)(*([tiles.data_ptr()] * gw.rows))
    assert call(0, 8, gg=gw, tbl=tw_) == TD_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert _same_bits(out, sent), "a refused call wrote the latent"


# ------------------------------------------------------------------------------------------------ 2. StripExchange, k ranks in one process
MOD_STRIP_RUNS = [("cfg2", "f16", k) for k in (2, 3, 5, 8)] + [("e", "bf16", 3), ("a", "f32", 4), ("d", "f16", 8), ("p4_32", "bf16", 5)]


@pytest.mark.parametrize("name,dn,world", MOD_STRIP_RUNS)
def test_mixture_strip_exchange_emulated_ranks(monkeypatch, name, dn, world):
    case = _row_case(name)
    N, C, W, H, tw, th, ov, bs = case[1]
    g, plan, _, _ = _mod_inputs(case, dn)
    dt = DTYPES[dn]
    ys = list(g.ys[:g.rows])
    torch.cuda.init()
    # the Mixture-of-Diffusers form: the latent buffer has the latent dtype
    monkeypatch.setattr(parallel, "StripExchange", functools.partial(parallel.StripExchange, latent_dtype=dt))
    shards, exs = _build_exchanges(monkeypatch, ys, g, N, C, dt, world)
    try:
        tw_d, rs_d = torch.from_numpy(plan.tile_weights).cuda(), torch.from_numpy(plan.rescale_factor).cuda()
        bboxes = [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)]
        for ex in exs:
            assert ex.x_out.dtype == dt
            ex.x_out.copy_(_sentinel(ex.x_out.shape, dt))
        for step in range(1, 4):
            _, _, x, _, _, _ = _inputs(case, dn, step)
            want_d = _mod_inputs(case, dn, step)[3].cuda()
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
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                first, count = _span({p for (_, p, _, _) in sh.halo_in()})
                raw = _raw_u32(ex.flags_tiles._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), _u32_at(raw, 128, 1)[0], f"{name} world {world} step {step}: blend of rank {r}", first)
                assert ex.blend_mixture(g, tw_d, rs_d) is ex.x_out
            for r in reversed(range(world)):
                sh, ex = shards[r], exs[r]
                first, count = _span({q for (q, _, _) in sh.x_in()})
                raw = _raw_u32(ex.flags_x._buf)
                _assert_ready(_u32_at(raw, 4 * first, count), (_u32_at(raw, 128, 1)[0] + P) & MASK,
                              f"{name} world {world} step {step}: latent-halo push of rank {r}", first)
                ex.push_x_halos_and_wait()
            torch.cuda.synchronize()
            union = _sentinel(want_d.shape, dt)
            for r, (sh, ex) in enumerate(zip(shards, exs)):
                lo, hi = sh.strip()
                for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]:
                    if b > a:
                        assert _same_bits(ex.x_out[:, :, a:b], want_d[:, :, a:b]), f"{name} {dn} world {world} step {step}: rank {r} rows [{a},{b})"
                union[:, :, lo:hi] = ex.x_out[:, :, lo:hi]
                for senders, fl, expect in (({p for (_, p, _, _) in sh.halo_in()}, ex.flags_tiles, P * (step + 1)),
                                            ({q for (q, _, _) in sh.x_in()}, ex.flags_x, P * step)):
                    raw = _raw_u32(fl._buf)
                    first, count = _span(senders)
                    signal = set(range(first, first + count))
                    assert _u32_at(raw, 0, world) == [P * step if q in signal else 0 for q in range(world)], f"slots of rank {r}, step {step}"
                    assert _u32_at(raw, 128, 1)[0] == expect, f"expect counter of rank {r}, step {step}"
            assert _same_bits(union, want_d), f"{name} {dn} world {world} step {step}: union of the strips"
    finally:
        torch.cuda.synchronize()
        for ex in exs:
            ex.close()


# ------------------------------------------------------------------------------------------------ 3. the delegate
_BG, _FG = "Background", "Foreground"
ROWS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", _BG, 0.2, -1),
        (True, 0.4, 0.3, 0.45, 0.6, "a dog", "", _FG, 0.3, 5),
        (True, 0.0, 0.5, 0.3, 0.5, "grass", "", _BG, 0.2, -1)]
SCENARIOS = [("grid only", [], True), ("background regions", [r for r in ROWS if r[7] == _BG], True),
             ("foreground region", ROWS, True), ("no background layer", ROWS, False)]


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _delegate(c, rows, bg):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers
    d = MixtureOfDiffusers(types.SimpleNamespace(width=c["W"] * 8, height=c["H"] * 8, sampler_name="Euler a", disable_extra_networks=True),
                           types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None),
                                                                                      image_cfg_scale=None, step=0)))
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
    if rows:
        d.init_custom_bbox({i: row for i, row in enumerate(rows)}, bg, False)
    d.init_done()
    return d


def _step(d, x, N):
    """One hijacked apply_model call (identity-like fake denoiser per tile, fake region denoiser)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    batches = d.local_batched_bboxes if d._shard is not None else d.batched_bboxes
    it = {"i": 0}

    def apply_model(x_tile, t, c_):
        bb = batches[it["i"]]
        it["i"] += 1
        return synth.fake_denoise(x_tile, bb, N)
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: synth.fake_region_denoise(x_tile, bbox_id)
    d.hook()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4, device=x.device)], "c_concat": [torch.zeros(N, 5, 1, 1, device=x.device)]}
    out = model.apply_model(x, torch.ones(N, device=x.device), cond).clone()
    d.unhook()
    return out


def _gpu_mod_strip_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    torch.cuda.set_device(rank)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        c = dict(N=2, C=4, W=128, H=96, tw=16, th=16, ov=8, bs=4)
        N = c["N"]
        host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=None))
        for dn in ("f16", "bf16"):
            xs = [synth.latent(70 + k, (N, c["C"], c["H"], c["W"]), DTYPES[dn]) for k in range(3)]
            for name, rows, bg in SCENARIOS:
                wants = [_step(_delegate(c, rows, bg), x.cuda(), N).cpu() for x in xs]      # the unsharded delegate
                d = _delegate(c, rows, bg)
                d.init_tile_shard(None, fused=True, mode="strip")
                assert d._shard_mode == "strip"
                for k, x in enumerate(xs):
                    out = _step(d, x.cuda(), N)
                    torch.cuda.synchronize()
                    what = f"rank {rank} {dn} {name} step {k}"
                    assert out.dtype == wants[k].dtype, f"{what}: returned {out.dtype}, the unsharded delegate {wants[k].dtype}"
                    lo, hi = d._strip.strip()
                    for (a, b) in [(lo, hi)] + [(a, b) for (_, a, b) in d._strip.x_in()]:
                        assert _same_bits(out[:, :, a:b].cpu(), wants[k][:, :, a:b]), f"{what}: rows [{a},{b})"
                    dist.barrier()
                    full = d.gather_latent(out)
                    assert _same_bits(full.cpu(), wants[k]), f"{what}: gathered latent"
                    dist.barrier()
                dist.barrier()
                d._strip_exchange.close()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


def test_one_rank_mixture_strip_delegate_bit_identical_to_unsharded(tmp_path):
    mp.spawn(_gpu_mod_strip_worker, args=(1, _free_port(), str(tmp_path)), nprocs=1, join=True)
    assert (tmp_path / "ok0").exists()


def test_multi_gpu_mixture_strip_delegate_bit_identical_to_one_gpu(tmp_path):
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs 2 GPUs")
    world = min(world, 4)
    mp.spawn(_gpu_mod_strip_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
