"""Model check of the row-strip exchange protocol (csrc/td_peer.cu td_push_regions + the in-kernel wait of
td_blend_multidiffusion_rows; parallel.StripExchange), no GPU: every rank is a little state machine whose micro-operations
(one CTA's data stores, one CTA's release add, one poll of a wait, one read of a halo) are interleaved at random.

Checked for many geometries / world sizes / schedules:
  * no deadlock: every rank finishes every step;
  * a blend reads, from every sender, exactly the halo of ITS step (never a stale one, never one overwritten by the
    sender's next step), and the next scatter reads the latent halo of its step;
  * a wait polls the contiguous slots [first, first + count) of StripShard.wait_range, which covers every rank that
    sends the waiter rows, and every rank in it pushes to the waiter once per step (StripShard.push_targets; a rank with
    no rows for it makes a signal-only push).
The model takes targets and wait ranges from the production bookkeeping instead of re-deriving them.
Per step and rank:  push_tiles (no counter of this rank touched)  ->  blend (wait: tile slots >= tile_expect)  ->
push_x (x_expect += P; push; wait: x slots >= x_expect; tile_expect += P).  tile_expect starts at P."""
import random

import pytest

from multidiffusion_upscaler_for_automatic1111_b200 import engine, parallel

P = 4          # CTAs per push in the model (TD_PUSH_CTAS = 32 on the device: only the count differs)


def _shards(W, H, tile, overlap, world):
    g = engine.make_grid(W, H, tile, tile, overlap, 4)
    return [parallel.StripShard(list(g.ys[:g.rows]), g.cols, g.tile_h, g.H, r, world) for r in range(world)]


def _rank_program(r, shards, state, steps):
    """Generator of micro-operations of rank r; yields after each one (True = progressed, False = polled and must retry)."""
    sh = shards[r]
    tile_data_targets = sorted({q for (_, q, _, _) in sh.halo_out()})
    tile_senders = sorted({p for (_, p, _, _) in sh.halo_in()})
    x_data_targets = sorted({p for (p, _, _) in sh.x_out()})
    x_senders = sorted({q for (q, _, _) in sh.x_in()})
    tile_targets, x_targets = sh.push_targets("tiles"), sh.push_targets("x")
    tile_wait, x_wait = sh.signallers("tiles"), sh.signallers("x")
    for kind, senders, wait in (("tiles", tile_senders, tile_wait), ("x", x_senders, x_wait)):
        assert set(senders) <= set(wait), f"rank {r}: {kind} senders {senders} outside the wait range {wait}"
    assert set(tile_data_targets) <= set(tile_targets) and set(x_data_targets) <= set(x_targets)
    for s in range(1, steps + 1):
        # scatter: reads the latent halo rows published at the end of step s - 1
        for q in x_senders:
            assert state["x_data"][r][q] == [s - 1] * P, f"rank {r} step {s}: scatter saw latent halo {state['x_data'][r][q]} from {q}"
            yield True
        # push_tiles: every CTA stores its share, then adds 1 (release) to each target's slot
        for cta in range(P):
            for q in tile_data_targets:
                state["tile_data"][q][r][cta] = s
                yield True
            for q in tile_targets:
                state["tile_slot"][q][r] += 1
                yield True
        # blend: the halo CTAs poll until every slot of the wait range has reached this rank's expect counter, then read
        want = state["tile_expect"][r]
        while any(state["tile_slot"][r][p] < want for p in tile_wait):
            yield False
        for p in tile_senders:
            yield True          # (other ranks may run between the wait and the read)
            assert state["tile_data"][r][p] == [s] * P, f"rank {r} step {s}: blend read halo {state['tile_data'][r][p]} of rank {p}"
        # push_x: bump own expect, push + signal, wait for own senders, then advance the tile set's expect counter
        state["x_expect"][r] += P
        yield True
        for cta in range(P):
            for q in x_data_targets:
                state["x_data"][q][r][cta] = s
                yield True
            for q in x_targets:
                state["x_slot"][q][r] += 1
                yield True
        while any(state["x_slot"][r][q] < state["x_expect"][r] for q in x_wait):
            yield False
        state["tile_expect"][r] += P
        yield True
    state["done"][r] = True


def _run(shards, steps, rng):
    world = len(shards)
    zeros = lambda: [[0] * world for _ in range(world)]
    state = {"tile_slot": zeros(), "x_slot": zeros(), "tile_expect": [P] * world, "x_expect": [0] * world,
             "tile_data": [[[0] * P for _ in range(world)] for _ in range(world)],
             "x_data": [[[0] * P for _ in range(world)] for _ in range(world)], "done": [False] * world}
    progs = [_rank_program(r, shards, state, steps) for r in range(world)]
    live = list(range(world))
    stalled = 0
    while live:
        r = rng.choice(live)
        burst = rng.choice((1, 1, 2, 5, 40))          # short and long time slices
        for _ in range(burst):
            try:
                progressed = next(progs[r])
            except StopIteration:
                live.remove(r)
                break
            stalled = 0 if progressed else stalled + 1
            if not progressed:
                break
        assert stalled < 20000 * world, f"deadlock: ranks {live} all polling, state {state['tile_slot']} / {state['tile_expect']}"
    assert all(state["done"])


# the last three have a tile pitch of 4 (overlap = tile - 4, the largest overlap the plan allows): from world 4 on, the
# latent-halo senders of a rank can skip a rank whose strip is empty
GEOMS = [(512, 512, 96, 48), (512, 1024, 96, 48), (256, 640, 64, 16), (128, 320, 96, 8),
         (16, 28, 16, 12), (32, 44, 32, 28), (96, 108, 96, 92)]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_strip_protocol_under_random_schedules(geom, world):
    W, H, tile, overlap = geom
    shards = _shards(W, H, tile, overlap, world)
    for seed in range(12):
        _run(shards, steps=4, rng=random.Random(1000 * world + seed))


def test_a_stale_expect_counter_would_be_caught():
    """The model is sharp: if the tile expect counter were advanced by the tile push itself (i.e. read by a concurrent blend
    before the bump), a blend could run on the previous step's halo -- emulate by starting tile_expect one push behind."""
    shards = _shards(512, 512, 96, 48, 2)
    global P
    with pytest.raises(AssertionError):
        for seed in range(200):
            rng = random.Random(seed)
            world = 2
            zeros = lambda: [[0] * world for _ in range(world)]
            state = {"tile_slot": zeros(), "x_slot": zeros(), "tile_expect": [0] * world, "x_expect": [0] * world,
                     "tile_data": [[[0] * P for _ in range(world)] for _ in range(world)],
                     "x_data": [[[0] * P for _ in range(world)] for _ in range(world)], "done": [False] * world}
            progs = [_rank_program(r, shards, state, 3) for r in range(world)]
            live = [0, 1]
            while live:
                r = rng.choice(live)
                try:
                    next(progs[r])
                except StopIteration:
                    live.remove(r)


def _check_flag_bookkeeping(sh, world, shards=None):
    """Every slot of a rank's wait range is signalled by its rank exactly once per step, the range covers every rank that
    sends the waiter rows, nobody pushes to a rank that does not poll its slot, and the range lies on the side that
    cannot close a wait cycle (tile halo: lower ranks; latent halo: higher ranks).  With `shards` (one per rank), every
    rank's own view must agree with `sh`'s."""
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    for kind in ("tiles", "x"):
        targets = [sh.push_targets(kind, q) for q in range(world)]
        for q in range(world):
            assert targets[q] == sorted(set(targets[q])) and q not in targets[q], f"{kind}: rank {q} targets {targets[q]}"
        for r in range(world):
            first, count = sh.wait_range(kind, r)
            if shards is not None:
                assert (first, count) == shards[r].wait_range(kind) and targets[r] == shards[r].push_targets(kind)
            assert 0 <= count <= _cabi.TD_MAX_PEERS and (count == 0 or 0 <= first and first + count <= world)
            wait = list(range(first, first + count))
            assert sh.signallers(kind, r) == wait
            senders = {p for (_, p, _, _) in sh.halo_in(r)} if kind == "tiles" else {q for (q, _, _) in sh.x_in(r)}
            assert senders <= set(wait), f"{kind}: rank {r} reads rows of {sorted(senders)} but waits on {wait}"
            assert all((q < r) if kind == "tiles" else (q > r) for q in wait), f"{kind}: rank {r} waits on {wait}"
            for q in range(world):      # pushes of one step that land in slot q of rank r: one per rank in the range
                n = targets[q].count(r)
                assert n == (1 if q in wait else 0), f"{kind}: slot {q} of rank {r} (wait range {wait}) is bumped by {n} pushes"


def test_smallest_latent_halo_range_with_a_silent_rank():
    """H = 28, tile 16, overlap 12, world 4: rank 0 reads latent rows of ranks 1 and 3; rank 2 owns an empty strip and has
    no rows for it, yet lies inside rank 0's wait range -- it must make a signal-only push to rank 0 every step."""
    shards = _shards(16, 28, 16, 12, 4)
    sh = shards[0]
    assert sh.ys == [0, 4, 8, 12] and sh.B == [0, 0, 8, 8, 28]
    assert sh.x_in(0) == [(1, 0, 8), (3, 8, 16)]
    assert sh.x_out(2) == []
    assert sh.wait_range("x", 0) == (1, 3)
    assert sh.x_in(1) == [(3, 8, 20)] and sh.push_targets("x", 2) == [0]
    _check_flag_bookkeeping(sh, 4, shards)


@pytest.mark.parametrize("tile,overlap", [(16, 12), (32, 28), (96, 92), (16, 8), (96, 88), (64, 16), (96, 48)])
def test_flag_bookkeeping_sweep(tile, overlap):
    """Deterministic sweep over tile pitches 4, 8 and 48 (and 48 at tile 64), canvas heights and worlds 1-16."""
    for H in range(tile, 4 * tile + 100, 4 if tile - overlap == 4 else 12):
        g = engine.make_grid(tile, H, tile, tile, overlap, 4)
        ys = list(g.ys[:g.rows])
        for world in range(1, 17):
            _check_flag_bookkeeping(parallel.StripShard(ys, g.cols, g.tile_h, g.H, 0, world), world)
