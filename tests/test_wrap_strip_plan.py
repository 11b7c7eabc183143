"""Row-strip tile shard on a periodic (seamless-tiling) plan, no GPU: parallel.StripShard(..., wrap_y=True) bookkeeping and the
flag protocol of the ring.

  * every canvas row has one owner; the tile halo a rank receives is exactly what its strip needs from foreign bands, across
    the seam included; the latent halo covers its modular scatter extent; blending each strip from own + received rows only
    (wrap_oracle) equals the whole-canvas wrapped step bit for bit, for MultiDiffusion and Mixture of Diffusers;
  * a plan wrapped in x only keeps the bounded plan's bookkeeping;
  * the exchange protocol with mirrored flag slots (slot r + world stands for rank r) under random schedules: no deadlock, no
    stale and no overwritten halo; a deterministic sweep of worlds 1-16 over the wait runs and push slots; and the model
    catches a sender that skips the mirrored slot."""
import random

import numpy as np
import pytest
import torch

import wrap_oracle as wo
from test_strip_protocol_model import P

from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel

WORLDS = [1, 2, 3, 4, 8, 12, 16]
# (W, H, tile, overlap, wrap): cfg2 wrapped in x and y; the 2048 x 512 panorama wrapped in x; a tile pitch of 4 wrapped in y
# (the last bands reach into several strips); tile == canvas; an odd canvas height wrapped in y
GEOMS = {"cfg2 xy": (512, 512, 96, 48, wo.WRAP_X | wo.WRAP_Y), "panorama x": (2048, 512, 96, 48, wo.WRAP_X),
         "pitch 4 y": (32, 44, 16, 12, wo.WRAP_Y), "tile == canvas xy": (64, 64, 64, 16, wo.WRAP_X | wo.WRAP_Y),
         "odd height y": (64, 75, 32, 16, wo.WRAP_Y)}


def _shards(W, H, tile, overlap, wrap, world):
    g = engine.make_grid(W, H, tile, tile, overlap, 4, wrap=wrap)
    ys = list(g.ys[:g.rows])
    return g, [parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world, wrap_y=bool(wrap & wo.WRAP_Y)) for r in range(world)]


def _band_rows(sh, i):
    """Canvas rows of band i (modular under wrap_y) -> {row: v}."""
    return {(sh.ys[i] + v) % sh.H if sh.wrap_y else sh.ys[i] + v: v for v in range(sh.tile_h)}


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", list(GEOMS))
def test_wrapped_strip_plan_covers_and_reproduces_the_single_device_blend(name, world):
    W, H, tile, ov, wrap = GEOMS[name]
    g, shards = _shards(W, H, tile, ov, wrap, world)
    plan = wo.WrapPlan(W, H, tile, tile, ov, 4, wrap, gaussian=True)
    assert [int(v) for v in g.ys[:g.rows]] == plan.ys and [int(v) for v in g.xs[:g.cols]] == plan.xs
    N, C, cols = 1, 2, g.cols
    x = torch.from_numpy(np.random.default_rng(world).standard_normal((N, C, H, W)).astype(np.float16))
    denoise = lambda t, bb: t * 0.5
    want_md, _ = wo.multidiffusion_step(x, plan, denoise)
    want_mod = wo.mixture_step(x, plan, denoise)
    tw, rs = torch.from_numpy(plan.tile_weights), torch.from_numpy(plan.rescale_factor).view(1, 1, H, W)
    wgt = torch.from_numpy(plan.weights).view(1, 1, H, W)
    outs = [denoise(wo.scatter(x, [b]), [b]) for b in plan.bboxes]
    got_md, got_mod = torch.full_like(want_md, float("nan")), torch.full_like(want_mod, float("nan"))
    owners = np.zeros(H, int)
    for r, sh in enumerate(shards):
        lo, hi = sh.strip()
        if hi <= lo:
            assert sh.halo_in() == []
            continue
        owners[lo:hi] += 1
        strip = set(range(lo, hi))
        # tile halo: exactly the strip rows of every foreign band that reaches the strip, one run of tile rows each
        got_halo = {i: (v0, v1) for (i, p, v0, v1) in sh.halo_in()}
        for (i, p, v0, v1) in sh.halo_in():
            assert sh.owner_of_band(i) == p and (i, r, v0, v1) in shards[p].halo_out()
        for i in range(sh.rows):
            if i in sh.bands():
                continue
            need = sorted(v for y, v in _band_rows(sh, i).items() if y in strip)
            if not need:
                assert i not in got_halo
                continue
            assert need == list(range(need[0], need[-1] + 1)) and got_halo[i] == (need[0], need[-1] + 1), f"rank {r} band {i}"
        # latent halo: the modular scatter extent of the own bands is strip + received rows
        have = np.zeros(H, bool)
        have[lo:hi] = True
        for (q, a, b) in sh.x_in():
            assert (r, a, b) in shards[q].x_out() and not have[a:b].any()
            have[a:b] = True
        for i in sh.bands():
            assert all(have[y] for y in _band_rows(sh, i)), f"rank {r}: latent halo misses rows of band {i}"
        # blend from own + received rows only: every other tile row is NaN
        avail = {i: (0, sh.tile_h) for i in sh.bands()}
        avail.update(got_halo)
        xb_md = torch.zeros((N, C, H, W), dtype=x.dtype)
        xb_mod = torch.zeros((N, C, H, W), dtype=x.dtype)
        for t, b in enumerate(plan.bboxes):
            i = t // cols
            if i not in avail:
                continue
            o = outs[t].clone()
            v0, v1 = avail[i]
            o[:, :, :v0] = float("nan")
            o[:, :, v1:] = float("nan")
            wo.accumulate_md(xb_md, o, [b], N)
            wo.accumulate_mod(xb_mod, o, [b], N, tw, rs)
        got_md[:, :, lo:hi] = wo.normalise_md(xb_md, wgt).float()[:, :, lo:hi]
        got_mod[:, :, lo:hi] = xb_mod[:, :, lo:hi]
    assert (owners == 1).all()
    assert torch.equal(got_md, want_md) and torch.equal(got_mod, want_mod)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("geom", [(2048, 512, 96, 48), (512, 512, 96, 48), (32, 44, 16, 12)])
def test_wrap_x_only_keeps_the_bounded_bookkeeping(geom, world):
    W, H, tile, ov = geom
    gw, wrapped = _shards(W, H, tile, ov, wo.WRAP_X, world)
    gb, bounded = _shards(W, H, tile, ov, 0, world)
    assert list(gw.ys[:gw.rows]) == list(gb.ys[:gb.rows])
    for a, b in zip(wrapped, bounded):
        assert not a.wrap_y and a.B == b.B and a.band_begin == b.band_begin and a.band_end == b.band_end
        assert a.halo_in() == b.halo_in() and a.halo_out() == b.halo_out() and a.scatter_rows() == b.scatter_rows()
        assert a.x_in() == b.x_in() and a.x_out() == b.x_out()
        for kind in ("tiles", "x"):
            assert a.wait_range(kind) == b.wait_range(kind) and a.push_targets(kind) == b.push_targets(kind)
            assert a.mirrored_targets(kind) == [] and a.push_slots(kind) == [(q, a.rank) for q in b.push_targets(kind)]


# ------------------------------------------------------------------------------------------------ flag protocol on the ring
def _ring_rank_program(r, shards, state, steps, mirror=True):
    """test_strip_protocol_model._rank_program with the ring's slots: a push bumps every (target, slot) of
    StripShard.push_slots (slot r, or r + world on a target that polls r in the wrapped part of its run), a wait polls the raw
    slots [first, first + count), up to 2 * world.  mirror=False bumps slot r everywhere instead."""
    sh, W = shards[r], len(shards)
    tile_data_targets = sorted({q for (_, q, _, _) in sh.halo_out()})
    tile_senders = sorted({p for (_, p, _, _) in sh.halo_in()})
    x_data_targets = sorted({p for (p, _, _) in sh.x_out()})
    x_senders = sorted({q for (q, _, _) in sh.x_in()})
    slots = {k: [(q, s if mirror else s % W) for (q, s) in sh.push_slots(k)] for k in ("tiles", "x")}
    wait = {k: range(sh.wait_range(k)[0], sum(sh.wait_range(k))) for k in ("tiles", "x")}
    for s in range(1, steps + 1):
        for q in x_senders:
            assert state["x_data"][r][q] == [s - 1] * P, f"rank {r} step {s}: scatter saw latent halo {state['x_data'][r][q]} from {q}"
            yield True
        for cta in range(P):
            for q in tile_data_targets:
                state["tile_data"][q][r][cta] = s
                yield True
            for (q, slot) in slots["tiles"]:
                state["tile_slot"][q][slot] += 1
                yield True
        want = state["tile_expect"][r]
        while any(state["tile_slot"][r][k] < want for k in wait["tiles"]):
            yield False
        for p in tile_senders:
            yield True
            assert state["tile_data"][r][p] == [s] * P, f"rank {r} step {s}: blend read halo {state['tile_data'][r][p]} of rank {p}"
        state["x_expect"][r] += P
        yield True
        for cta in range(P):
            for q in x_data_targets:
                state["x_data"][q][r][cta] = s
                yield True
            for (q, slot) in slots["x"]:
                state["x_slot"][q][slot] += 1
                yield True
        while any(state["x_slot"][r][k] < state["x_expect"][r] for k in wait["x"]):
            yield False
        state["tile_expect"][r] += P
        yield True
    state["done"][r] = True


def _ring_run(shards, steps, rng, mirror=True):
    world = len(shards)
    slots = lambda: [[0] * (2 * world) for _ in range(world)]
    state = {"tile_slot": slots(), "x_slot": slots(), "tile_expect": [P] * world, "x_expect": [0] * world,
             "tile_data": [[[0] * P for _ in range(world)] for _ in range(world)],
             "x_data": [[[0] * P for _ in range(world)] for _ in range(world)], "done": [False] * world}
    progs = [_ring_rank_program(r, shards, state, steps, mirror) for r in range(world)]
    live = list(range(world))
    stalled = 0
    while live:
        r = rng.choice(live)
        for _ in range(rng.choice((1, 1, 2, 5, 40))):
            try:
                progressed = next(progs[r])
            except StopIteration:
                live.remove(r)
                break
            stalled = 0 if progressed else stalled + 1
            if not progressed:
                break
        assert stalled < 20000 * world, f"deadlock: ranks {live} all polling"
    assert all(state["done"])


RING_GEOMS = [(512, 512, 96, 48), (64, 44, 16, 12), (32, 28, 16, 12), (64, 75, 32, 16), (96, 108, 96, 92)]


@pytest.mark.parametrize("geom", RING_GEOMS)
@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_ring_protocol_under_random_schedules(geom, world):
    W, H, tile, ov = geom
    _, shards = _shards(W, H, tile, ov, wo.WRAP_X | wo.WRAP_Y, world)
    for seed in range(8):
        _ring_run(shards, steps=4, rng=random.Random(7000 * world + seed))


def test_the_model_catches_a_missing_mirror_bump():
    """A pitch-4 plan wrapped in y, world 4: some wait runs wrap (e.g. ranks {3, 0} polled as slots 3, 4); they are never
    satisfied when the sender publishes into slot 0 instead of its mirror, slot 4."""
    _, shards = _shards(64, 44, 16, 12, wo.WRAP_Y, 4)
    assert any(sh.mirrored_targets(k) for sh in shards for k in ("tiles", "x")), "the geometry must exercise a mirrored slot"
    with pytest.raises(AssertionError, match="deadlock"):
        _ring_run(shards, steps=3, rng=random.Random(1), mirror=False)


def _check_ring_bookkeeping(shards):
    W = len(shards)
    for kind in ("tiles", "x"):
        for r, sh in enumerate(shards):
            first, count = sh.wait_range(kind)
            run = [k % W for k in range(first, first + count)]
            assert 0 <= count <= _cabi.TD_MAX_PEERS and (count == 0 or (0 <= first < W and first + count <= 2 * W <= 32))
            assert r not in run and len(set(run)) == len(run), f"{kind}: rank {r} waits on {run}"
            senders = {p for (_, p, _, _) in sh.halo_in()} if kind == "tiles" else {q for (q, _, _) in sh.x_in()}
            assert senders <= set(run), f"{kind}: rank {r} reads rows of {sorted(senders)} but waits on {run}"
            for slot in range(first, first + count):      # every slot of the run is bumped once per step by its rank
                bumps = [(p, s) for p in range(W) for (q, s) in shards[p].push_slots(kind) if q == r and s == slot]
                assert bumps == [(slot % W, slot)], f"{kind}: slot {slot} of rank {r} is bumped by {bumps}"
        for p, sh in enumerate(shards):
            assert len(sh.push_slots(kind)) <= _cabi.TD_MAX_PEERS, f"{kind}: rank {p} publishes into {sh.push_slots(kind)}"
            for (q, s) in sh.push_slots(kind):                # ... and nobody bumps a slot its target does not poll ...
                first, count = shards[q].wait_range(kind)
                assert s % W == p and first <= s < first + count, f"{kind}: rank {p} bumps slot {s} of {q} (run {first}+{count})"
    # ... and no halo is overwritten while it is read: a rank that sends tile halo to q waits for q's latent push
    for p, sh in enumerate(shards):
        for (_, q, _, _) in sh.halo_out():
            assert q in {s for (s, _, _) in sh.x_in()}, f"rank {p} sends tile halo to {q} but reads no latent rows of it"


@pytest.mark.parametrize("tile,overlap", [(16, 12), (32, 28), (96, 92), (16, 8), (96, 88), (64, 16), (96, 48)])
def test_ring_bookkeeping_sweep(tile, overlap):
    """Deterministic sweep over tile pitches 4, 8 and 48 (and 48 at tile 64), canvas heights and worlds 1-16, wrapped in y."""
    for H in range(tile, 4 * tile + 100, 4 if tile - overlap == 4 else 12):
        for world in range(1, 17):
            _, shards = _shards(tile, H, tile, overlap, wo.WRAP_Y, world)
            _check_ring_bookkeeping(shards)


def test_one_rank_ring_has_no_halo():
    _, (sh,) = _shards(512, 512, 96, 48, wo.WRAP_X | wo.WRAP_Y, 1)
    assert sh.halo_in() == [] and sh.x_in() == [] and sh.strip() == (0, 512)
    for kind in ("tiles", "x"):
        assert sh.wait_range(kind) == (0, 0) and sh.push_slots(kind) == []


def test_seam_halo_goes_from_the_last_rank_to_rank_0():
    _, shards = _shards(512, 512, 96, 48, wo.WRAP_X | wo.WRAP_Y, 2)
    last = shards[0].rows - 1
    assert shards[0].ys[last] + 96 > 512
    assert (last, 1, 512 - shards[0].ys[last], 96) in shards[0].halo_in()
    assert shards[1].scatter_spans()[0][0] == 0 and any(q == 0 and a == 0 for (q, a, b) in shards[1].x_in())
    assert shards[0].wait_range("tiles") == (1, 1) and shards[1].wait_range("tiles") == (0, 1)
