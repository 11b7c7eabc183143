"""Region prompt control (custom bboxes) under the multi-GPU tile shard.

CPU: the ownership / packing plan of parallel.RegionShard; the sharded MultiDiffusion and Mixture of Diffusers delegates
with regions on gloo processes (device kernels swapped for the oracle) against the single-process oracle; and a simulation
of the row-strip shard's region exchange and per-strip composite against the whole-canvas composite.
GPU: td_region_composite_rows against td_region_composite, and (two or more GPUs) the sharded delegates with regions
against a single-GPU run, bit for bit."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import DTYPES, assert_bit_equal, region_composite_reference
from oracle import blend, region, synth, tiling

_BG, _FG = "Background", "Foreground"

# canvas W x H = 64 x 48 latent pixels, 16-pixel tiles with overlap 8 (5 x 7 = 35 tiles)
GRID = dict(N=2, C=4, W=64, H=48, tw=16, th=16, ov=8, bs=4)
ROWS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", _BG, 0.2, -1),
        (True, 0.4, 0.3, 0.45, 0.6, "a dog", "", _FG, 0.3, 5),
        (True, 0.0, 0.5, 0.3, 0.5, "grass", "", _BG, 0.2, -1),
        (True, 0.55, 0.05, 0.4, 0.7, "a bird", "", _FG, 0.8, 7),
        (True, 0.2, 0.0, 0.6, 0.25, "sky", "", _FG, 0.5, 1)]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _init(rank, world, port, backend):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group(backend, rank=rank, world_size=world)


# ------------------------------------------------------------------------------------------------ plan (no GPU)
def _rects(k, H=48, W=64, seed=0):
    g = torch.Generator().manual_seed(seed + k)
    out = []
    for _ in range(k):
        y = int(torch.randint(0, H - 1, (1,), generator=g))
        x = int(torch.randint(0, W - 1, (1,), generator=g))
        out.append((x, y, int(torch.randint(1, W - x + 1, (1,), generator=g)), int(torch.randint(1, H - y + 1, (1,), generator=g))))
    return out


@pytest.mark.parametrize("world", range(1, 9))
def test_region_plan_owns_every_region_once_and_round_trips(world):
    from multidiffusion_upscaler_for_automatic1111_b200 import parallel
    N, C, H, W = 2, 3, 48, 64
    for k in (1, 3, 7, 13):
        rects = _rects(k)
        shards = [parallel.RegionShard(rects, r, world) for r in range(world)]
        assert all(s.owner == shards[0].owner for s in shards), "ownership differs between ranks"
        owned = sorted(j for r in range(world) for j in shards[0].mine(r))
        assert owned == list(range(k)), "a region is denoised zero or several times"
        assert all(shards[r].mine() == shards[0].mine(r) for r in range(world))

        # outputs: every rank's pack -> all-gather (stacked here) -> every region's output, bit-exact, on every rank
        outs = [synth.latent(100 + j, (N, C, h, w), torch.float16) for j, (_, _, w, h) in enumerate(rects)]
        like = torch.empty((N, C, H, W), dtype=torch.float16)
        packs = [s.pack_outputs([outs[j] for j in s.mine()], N * C, like) for s in shards]
        assert len({p.numel() for p in packs}) == 1
        gathered = torch.stack(packs)
        for s in shards:
            got = s.unpack_outputs(gathered, N, C)
            assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(got, outs))

        # inputs: strips of a monotone partition of the rows; each rank packs only its own rows
        B = sorted(int(v) for v in torch.randint(0, H + 1, (world - 1,), generator=torch.Generator().manual_seed(k)))
        B = [0] + B + [H]
        x = synth.latent(7, (N, C, H, W), torch.bfloat16)
        packs = []
        for r, s in enumerate(shards):
            xr = torch.full_like(x, float("nan"))           # rows outside the strip are not valid on rank r
            xr[:, :, B[r]:B[r + 1]] = x[:, :, B[r]:B[r + 1]]
            packs.append(s.pack_inputs(xr, B))
        gathered = torch.stack(packs)
        for s in shards:
            ins = s.unpack_inputs(gathered, B, N, C)
            assert sorted(ins) == s.mine()
            for j, t in ins.items():
                rx, ry, w, h = rects[j]
                assert torch.equal(t.view(torch.int16), x[:, :, ry:ry + h, rx:rx + w].contiguous().view(torch.int16))


@pytest.mark.parametrize("world", [1, 3])
def test_region_output_exchange_carries_every_output_dtype_exactly(world, monkeypatch):
    """The exchange packs fp32 whatever the latent dtype, so fp16, bf16 and fp32 outputs all reach the composite as the UNet
    returned them; a pack that would round an output (fp32 into fp16, fp16 into bf16) is refused."""
    from multidiffusion_upscaler_for_automatic1111_b200 import parallel
    N, C, H, W = 2, 3, 48, 64
    rects = _rects(5)
    shards = [parallel.RegionShard(rects, r, world) for r in range(world)]
    like = torch.empty((N, C, H, W), dtype=torch.float16)
    for odt in (torch.float16, torch.bfloat16, torch.float32):
        # values with more significant bits than fp16 / bf16 keep, before the cast to odt
        outs = [synth.latent(100 + j, (N, C, h, w), torch.float32).mul_(1.0 + 2 ** -20).to(odt) for j, (_, _, w, h) in enumerate(rects)]
        packs = [s.pack_outputs([outs[j] for j in s.mine()], N * C, like, torch.float32) for s in shards]
        assert all(p.dtype == torch.float32 for p in packs)
        def all_gather(local, group=None):       # every rank's pack, as the collective returns them
            assert local.dtype == torch.float32 and local.numel() == packs[0].numel()
            return torch.stack(packs)
        monkeypatch.setattr(parallel, "gather_tile_outputs", all_gather)
        for s in shards:
            got = parallel.exchange_region_outputs(s, [outs[j] for j in s.mine()], like)
            assert all(a.dtype == torch.float32 and torch.equal(a, b.float()) and torch.equal(a.to(odt).view(torch.uint8), b.view(torch.uint8))
                       for a, b in zip(got, outs)), odt
    mine = shards[0].mine()
    f32 = [synth.latent(7, (N, C, rects[j][3], rects[j][2]), torch.float32) for j in mine]
    with pytest.raises(ValueError, match="does not fit"):
        shards[0].pack_outputs(f32, N * C, like)
    with pytest.raises(ValueError, match="does not fit"):
        shards[0].pack_outputs([o.half() for o in f32], N * C, like, torch.bfloat16)


# ------------------------------------------------------------------------------------------------ strip simulation (no GPU)
# canvas 48 x 120, tiles 16 / overlap 8: 14 tile rows; at 6 ranks the strips are [0,24) [24,48) [48,64) [64,80) [80,96) [96,120)
STRIP_GEOM = dict(W=48, H=120, tw=16, th=16, ov=8)
STRIP_LAYOUTS = {
    "inside_one_strip": [(4, 2, 20, 10, 0)],
    "crossing_one_boundary": [(0, 40, 30, 16, 1)],
    "crossing_two_boundaries": [(10, 20, 30, 50, 0), (3, 44, 20, 30, 1)],
    "touching_last_row": [(5, 100, 40, 20, 1), (0, 112, 48, 8, 0)],
    "overlapping_foregrounds": [(0, 10, 40, 60, 1), (8, 30, 40, 70, 1), (20, 50, 20, 20, 1), (0, 0, 48, 120, 0)],
}


@pytest.mark.parametrize("world", range(1, 7))
@pytest.mark.parametrize("layout", list(STRIP_LAYOUTS))
@pytest.mark.parametrize("method", ["md", "mod"])
def test_strip_region_exchange_and_row_composites_reproduce_the_whole_canvas(world, layout, method):
    """Rank r holds the latent and the grid accumulator only on its strip [B_r, B_{r+1}); it packs the region rows of its
    strip, denoises the regions it owns from the gathered rows, and composites its own rows from the gathered outputs.
    The union of the strips must equal the whole-canvas composite bit for bit."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine, parallel
    c = STRIP_GEOM
    N, C, H, W = 2, 4, c["H"], c["W"]
    g = engine.make_grid(W, H, c["tw"], c["th"], c["ov"], 4)
    ys = list(g.ys[:g.rows])
    strips = [parallel.StripShard(ys, g.cols, c["th"], H, r, world) for r in range(world)]
    B = strips[0].B
    rects = STRIP_LAYOUTS[layout]
    if world == 6:      # the layouts do what their names say
        assert B == [0, 24, 48, 64, 80, 96, 120]
        most = max(sum(1 for b in B[1:-1] if y < b < y + h) for (_, y, _, h, _) in rects)
        assert most == {"inside_one_strip": 0, "crossing_one_boundary": 1}.get(layout, most) and (most >= 2 or "two" not in layout)
        assert any(y + h == H for (_, y, _, h, _) in rects) or layout != "touching_last_row"
    gen = torch.Generator().manual_seed(world * 31 + len(layout))
    x = synth.latent(3, (N, C, H, W), torch.float16)
    acc = (torch.randn((N, C, H, W), generator=gen) * 2).to(torch.float16)          # grid accumulator (un-normalised)
    weights = torch.randint(0, 5, (H, W), generator=gen).float() if method == "md" else None
    aux = []
    for (_, _, w, h, mode) in rects:
        if mode == 1:
            aux.append(torch.rand((h, w), generator=gen))
        else:
            aux.append(None if method == "md" else torch.rand((1, 1, h, w), generator=gen) * 3)

    def denoise(t, j):
        return synth.fake_region_denoise(t, j)

    full_regions = [(rx, ry, w, h, m, denoise(x[:, :, ry:ry + h, rx:rx + w], j), aux[j]) for j, (rx, ry, w, h, m) in enumerate(rects)]
    want = region_composite_reference(acc, weights, full_regions)

    shards = [parallel.RegionShard([r[:4] for r in rects], r, world) for r in range(world)]
    invalid = lambda t, lo, hi: torch.cat([torch.full_like(t[:, :, :lo], float("nan")), t[:, :, lo:hi],
                                           torch.full_like(t[:, :, hi:], float("nan"))], dim=2)
    gathered_in = torch.stack([s.pack_inputs(invalid(x, B[r], B[r + 1]), B) for r, s in enumerate(shards)])
    packs = []
    for s in shards:
        ins = s.unpack_inputs(gathered_in, B, N, C)
        packs.append(s.pack_outputs([denoise(ins[j], j) for j in s.mine()], N * C, x))
    gathered_out = torch.stack(packs)
    got = torch.full((N, C, H, W), float("nan"))
    for r, s in enumerate(shards):
        lo, hi = strips[r].strip()
        outs = s.unpack_outputs(gathered_out, N, C)
        regions_r = [(rx, ry, w, h, m, outs[j], aux[j]) for j, (rx, ry, w, h, m) in enumerate(rects)]
        o = region_composite_reference(invalid(acc, lo, hi), weights, regions_r)
        got[:, :, lo:hi] = o[:, :, lo:hi]
    assert_bit_equal(got, want, f"{layout} world {world}")


# ------------------------------------------------------------------------------------------------ gloo delegates (no GPU)
def _install_oracle_engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200.tile_methods import abstractdiffusion

    def bbs(g):
        return [tuple(int(v) for v in r) for r in engine.grid_bboxes_xywh(g)]

    def scatter_tiles(g, x, out=None, tile_begin=0, tile_end=None, flags=0):
        return blend.scatter_tiles(x, bbs(g)[tile_begin:tile_end])

    def blend_multidiffusion(g, outs, N, C, tile_bs, weights, acc_dtype, x_buffer=None, flags=0, out=None, rcp_weights=None):
        buf = torch.zeros((N, C, g.H, g.W), dtype=acc_dtype)
        blend.accumulate_md(buf, torch.cat(list(outs), dim=0), bbs(g), N)
        if x_buffer is not None:
            x_buffer.copy_(buf)
        return blend.normalise_md(buf, weights.to(buf.device))

    def blend_mixture(g, outs, N, C, tile_bs, tile_weights, rescale, x_buffer, flags=0):
        x_buffer.zero_()
        blend.accumulate_mod(x_buffer, torch.cat(list(outs), dim=0), bbs(g), N, tile_weights.to(x_buffer.device), rescale.to(x_buffer.device))
        return x_buffer

    engine.scatter_tiles, engine.blend_multidiffusion, engine.blend_mixture = scatter_tiles, blend_multidiffusion, blend_mixture
    engine.region_composite = region_composite_reference
    abstractdiffusion.AbstractDiffusion._check_input = lambda self, x: x.contiguous()


def _p(c):
    return types.SimpleNamespace(width=c["W"] * 8, height=c["H"] * 8, sampler_name="Euler a", disable_extra_networks=True)


def _sampler():
    return types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None,
                                                                      step=0))


def _oracle_step(method, x, bg, rows):
    c = GRID
    N = x.shape[0]
    plan = tiling.GridPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], method == "mod")
    regs = region.make_regions(rows, c["W"], c["H"])
    w = region.weights_with_regions(plan.weights if bg else None, regs, c["H"], c["W"], method)
    den = lambda t, bb: synth.fake_denoise(t, bb, N)
    if method == "md":
        return region.multidiffusion_region_step(x, plan.batched_bboxes, w, regs, den, synth.fake_region_denoise, bg)
    return region.mixture_region_step(x, plan.batched_bboxes, plan.tile_weights, w, regs, den, synth.fake_region_denoise, bg)


def _delegate(method, bg, with_grid, calls, fused=False, rows=ROWS):
    # fused=False: the replicate mode over an all-gather (the strip and peer-memory forms need CUDA IPC)
    """A sharded delegate with ROWS; its region denoiser records (bbox_id) into `calls`.  Returns (delegate, step(x))."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    c = GRID
    N = c["N"]

    def custom(x_tile, bbox_id, bbox):
        calls.append(bbox_id)
        return synth.fake_region_denoise(x_tile, bbox_id)

    cls = MultiDiffusion if method == "md" else MixtureOfDiffusers
    d = cls(_p(c), _sampler())
    if with_grid:
        d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
    if rows:
        d.init_custom_bbox({i: row for i, row in enumerate(rows)}, bg, False)
    d.init_done()
    d.init_tile_shard(None, fused=fused)
    if method == "md":
        def step(x):
            return d.sample_one_step(x, None, lambda t, bb: synth.fake_denoise(t, bb, N), custom)
        return d, step
    it = {"i": 0}

    def apply_model(x_tile, t, c_):
        bb = d.local_batched_bboxes[it["i"]]
        it["i"] += 1
        return synth.fake_denoise(x_tile, bb, N)
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: custom(x_tile, bbox_id, bbox)
    d.hook()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4)], "c_concat": [torch.zeros(N, 5, 1, 1)]}

    def step(x):
        it["i"] = 0
        return model.apply_model(x, torch.ones(N), cond).clone()
    return d, step


def _gloo_region_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, host
    _install_oracle_engine()
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        for method in ("md", "mod"):
            for bg, with_grid in ((True, True), (False, True), (False, False)):
                state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
                host.use_shared(types.SimpleNamespace(state=state, sd_model=None))
                calls = []
                d, step = _delegate(method, bg, with_grid, calls)
                assert len(d.custom_bboxes) == len(ROWS)
                for k in range(3):
                    x = synth.latent(40 + k, (c["N"], c["C"], c["H"], c["W"]), torch.float16 if k != 1 else torch.float32)
                    del calls[:]
                    got = step(x)
                    want = _oracle_step(method, x, bg, ROWS)
                    assert torch.equal(got, want) and got.dtype == want.dtype, f"rank {rank} {method} bg={bg} grid={with_grid} step {k} differs"
                    everyone = [None] * world
                    dist.all_gather_object(everyone, list(calls))
                    assert sorted(j for cl in everyone for j in cl) == list(range(len(ROWS))), f"region calls per step: {everyone}"
                # an interrupt on the last rank: it still joins every exchange and returns its input; the next step is exact again
                state.interrupted = rank == world - 1
                x = synth.latent(50, (c["N"], c["C"], c["H"], c["W"]), torch.float16)
                got = step(x)
                if state.interrupted and (method == "md" or bg):      # Mixture of Diffusers polls only between grid batches
                    assert got is x or torch.equal(got, x), f"{method} bg={bg} grid={with_grid}: the interrupted rank did not return its input"
                state.interrupted = False
                got = step(x)
                assert torch.equal(got, _oracle_step(method, x, bg, ROWS)), f"rank {rank} {method}: not in lock-step after an interrupt"
                if method == "mod":
                    MixtureOfDiffusers.unhook()
                host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_sharded_delegates_with_regions_equal_single(tmp_path, world):
    mp.spawn(_gloo_region_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


_K = torch.tensor(0.7071, dtype=torch.float32)      # fp32 UNet stand-ins: outputs with more bits than the fp16 latent


def _f32_denoise(t, bb, N):
    return synth.fake_denoise(t.float(), bb, N) * _K


def _f32_region_denoise(t, j):
    return synth.fake_region_denoise(t.float(), j) * _K


def _oracle_step_f32(method, x, bg, rows, region_denoise=_f32_region_denoise):
    c = GRID
    N = x.shape[0]
    plan = tiling.GridPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], method == "mod")
    regs = region.make_regions(rows, c["W"], c["H"])
    w = region.weights_with_regions(plan.weights if bg else None, regs, c["H"], c["W"], method)
    den = lambda t, bb: _f32_denoise(t, bb, N)
    if method == "md":
        return region.multidiffusion_region_step(x, plan.batched_bboxes, w, regs, den, region_denoise, bg)
    return region.mixture_region_step(x, plan.batched_bboxes, plan.tile_weights, w, regs, den, region_denoise, bg)


def _gloo_f32_unet_worker(rank, world, port, result_dir, n_rows):
    """A UNet that returns fp32 for an fp16 latent, sharded: the region outputs cross the all-gather as the UNet returned
    them (also from and to a rank that owns no region), so every rank composites what one process composites."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    _install_oracle_engine()
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = c["N"]
        rows = ROWS[:n_rows]
        for method in ("md", "mod"):
            for bg in (True, False):
                host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1),
                                                      sd_model=None))
                d = (MultiDiffusion if method == "md" else MixtureOfDiffusers)(_p(c), _sampler())
                d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
                d.init_custom_bbox({i: row for i, row in enumerate(rows)}, bg, False)
                d.init_done()
                d.init_tile_shard(None, fused=False)
                x = synth.latent(45, (N, c["C"], c["H"], c["W"]), torch.float16)
                if method == "md":
                    got = d.sample_one_step(x, None, lambda t, bb: _f32_denoise(t, bb, N), lambda t, j, b: _f32_region_denoise(t, j))
                else:
                    it = {"i": 0}

                    def apply_model(x_tile, t, c_):
                        bb = d.local_batched_bboxes[it["i"]]
                        it["i"] += 1
                        return _f32_denoise(x_tile, bb, N)
                    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt",
                                                  model=types.SimpleNamespace(conditioning_key="crossattn"))
                    host.get_shared().sd_model = model
                    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: _f32_region_denoise(x_tile, bbox_id)
                    d.hook()
                    got = model.apply_model(x, torch.ones(N), {"c_crossattn": [torch.zeros(N, 2, 4)], "c_concat": [torch.zeros(N, 5, 1, 1)]})
                    MixtureOfDiffusers.unhook()
                want = _oracle_step_f32(method, x, bg, rows)
                assert got.dtype == want.dtype and torch.equal(got.view(torch.uint8), want.view(torch.uint8)), \
                    f"rank {rank} {method} bg={bg}: sharded step with fp32 region outputs differs from one process"
                # outputs rounded to the latent dtype before the add give another result (not without a background: the
                # first add into zeros is that rounding)
                rounded = _oracle_step_f32(method, x, bg, rows, lambda t, j: _f32_region_denoise(t, j).to(t.dtype))
                assert not bg or not torch.equal(rounded, want), f"{method}: rounding the region outputs first changes nothing"
                host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n_rows", [(2, len(ROWS)), (3, 2)])
def test_gloo_sharded_delegates_with_fp32_region_outputs_equal_single(tmp_path, world, n_rows):
    """(3, 2): rank 2 owns no region and still packs and receives fp32."""
    mp.spawn(_gloo_f32_unet_worker, args=(world, _free_port(), str(tmp_path), n_rows), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


def _gloo_noise_worker(rank, world, port, result_dir):
    """Noise inversion's tiled eps prediction (`get_noise`, both delegates) with regions: sharded == one process."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils import utils
    _install_oracle_engine()
    utils.Condition.reconstruct_cond = staticmethod(lambda cond, step: cond.clone())
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = 1

        def apply_model(x, sigma, cond=None):        # scale by the first text-cond value: regions (cond j + 1) differ from tiles
            t = cond["c_crossattn"]
            t = t[0] if isinstance(t, list) else t
            return (x.float() * (0.5 + 0.25 * float(t.flatten()[0]))).to(x.dtype)
        model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
        host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=model))
        x = synth.latent(70, (N, c["C"], c["H"], c["W"]), torch.float32)
        cond = {"c_crossattn": [torch.zeros(N, 2, 4)], "c_concat": [torch.zeros(N, 5, 1, 1)]}
        for cls in (MultiDiffusion, MixtureOfDiffusers):
            res = []
            for shard in (False, True):
                d = cls(_p(c), _sampler())
                d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
                d.init_custom_bbox({i: row for i, row in enumerate(ROWS)}, True, False)
                d.init_done()
                for j, b in enumerate(d.custom_bboxes):
                    b.cond = torch.full((2, 4), float(j + 1))
                if shard:
                    d.init_tile_shard(None, fused=False)
                if cls is MixtureOfDiffusers:
                    d.hook()
                res.append(d.get_noise(x, torch.ones(N), cond, 3).clone())
                if cls is MixtureOfDiffusers:
                    MixtureOfDiffusers.unhook()
            assert torch.equal(res[0], res[1]), f"rank {rank} {cls.__name__}: sharded get_noise differs"
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


def test_gloo_sharded_noise_inversion_eps_with_regions_equals_single(tmp_path):
    mp.spawn(_gloo_noise_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()


class _OracleStripExchange:
    """parallel.StripExchange's interface on CPU tensors over gloo, so that MultiDiffusion's strip tail (`_strip_step`) runs
    without CUDA IPC: the tile outputs of all ranks are all-gathered and the oracle blends the OWN rows only; the latent halo
    and `gather_latent` move strips with all-gathers.  Rows a rank does not own or receive stay NaN."""

    def __init__(self, d, N, C, dtype):
        self.d, self.sh, self.N, self.C, self.dtype = d, d._strip, N, C, dtype
        self.x_out = torch.full((N, C, d.h, d.w), float("nan"))
        self.blends = 0

    def own_tiles(self):
        t0, t1 = self.sh.tile_range()
        self._own = torch.empty(((t1 - t0) * self.N, self.C, self.sh.tile_h, self.d.tile_w), dtype=self.dtype)
        return self._own

    def push_tile_halos(self):
        pass

    def blend(self, g, weights, rcp_weights, flags=0, x_buffer=None):
        from multidiffusion_upscaler_for_automatic1111_b200 import engine
        sh, N = self.sh, self.N
        most = max(sh.tile_range(r)[1] - sh.tile_range(r)[0] for r in range(sh.world)) * N
        pad = torch.zeros((most,) + tuple(self._own.shape[1:]), dtype=self.dtype)
        pad[:self._own.shape[0]] = self._own
        parts = [torch.empty_like(pad) for _ in range(sh.world)]
        dist.all_gather(parts, pad)
        tiles = torch.cat([parts[r][:(sh.tile_range(r)[1] - sh.tile_range(r)[0]) * N] for r in range(sh.world)])
        acc = torch.zeros((N, self.C, g.H, g.W), dtype=self.dtype)
        blend.accumulate_md(acc, tiles, [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)], N)
        lo, hi = sh.strip()
        self.x_out[:, :, lo:hi] = blend.normalise_md(acc, weights.cpu())[:, :, lo:hi]
        if x_buffer is not None:
            x_buffer[:, :, lo:hi] = acc[:, :, lo:hi]
        self.blends += 1
        return self.x_out

    def _strips(self, x):
        sh = self.sh
        rows = max(sh.B[r + 1] - sh.B[r] for r in range(sh.world))
        send = torch.zeros((x.shape[0], x.shape[1], rows, x.shape[3]), dtype=x.dtype)
        lo, hi = sh.strip()
        send[:, :, :hi - lo] = x[:, :, lo:hi]
        parts = [torch.empty_like(send) for _ in range(sh.world)]
        dist.all_gather(parts, send)
        return parts

    def push_x_halos_and_wait(self):
        parts = self._strips(self.x_out)
        for (q, a, b) in self.sh.x_in():
            self.x_out[:, :, a:b] = parts[q][:, :, a - self.sh.B[q]:b - self.sh.B[q]]

    def gather_latent(self, x):
        parts = self._strips(x)
        out = torch.empty_like(x)
        for r in range(self.sh.world):
            a, b = self.sh.strip(r)
            out[:, :, a:b] = parts[r][:, :, :b - a]
        return out


def _gloo_strip_worker(rank, world, port, result_dir):
    """MultiDiffusion's strip shard with regions through the delegate (`_sample_one_step_sharded` -> `_region_pass_sharded` ->
    `_strip_step` -> `_composite_regions(rows=...)`), on gloo with the exchange of _OracleStripExchange and the device kernels
    swapped for the oracle.  Each rank's input is valid only on its strip and latent halo; its own rows, its halo rows and the
    gathered latent must equal the single-process oracle, every step, also after an interrupt on one rank."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion, engine, host
    _install_oracle_engine()
    composites = []

    def region_composite_rows(x_buffer, weights, regions, row_begin, row_end, out):
        assert out.dtype == torch.float32 and tuple(out.shape) == tuple(x_buffer.shape), "the composite must write the latent buffer"
        composites.append((row_begin, row_end))
        out[:, :, row_begin:row_end] = region_composite_reference(x_buffer, weights, regions)[:, :, row_begin:row_end]
        return out
    engine.region_composite_rows = region_composite_rows
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = c["N"]
        for bg in (True, False):
            state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
            host.use_shared(types.SimpleNamespace(state=state, sd_model=None))
            calls = []

            def custom(x_tile, bbox_id, bbox):
                calls.append(bbox_id)
                return synth.fake_region_denoise(x_tile, bbox_id)
            d = MultiDiffusion(_p(c), _sampler())
            d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
            d.init_custom_bbox({i: row for i, row in enumerate(ROWS)}, bg, False)
            d.init_done()
            d.init_tile_shard(None, fused=True)
            assert d._shard_mode == "strip"
            sh = d._strip
            d._strip_exchange = ex = _OracleStripExchange(d, N, c["C"], torch.float16)
            lo, hi = sh.strip()
            valid = [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]
            for k in range(4):
                x = synth.latent(80 + k, (N, c["C"], c["H"], c["W"]), torch.float16)
                want = _oracle_step("md", x, bg, ROWS)
                x_r = torch.full_like(x, float("nan"))        # what this rank holds: its strip and latent halo
                for (a, b) in valid:
                    x_r[:, :, a:b] = x[:, :, a:b]
                state.interrupted = k == 2 and rank == world - 1
                del calls[:], composites[:]
                got = d.sample_one_step(x_r, None, lambda t, bb: synth.fake_denoise(t, bb, N), custom)
                assert composites == [(lo, hi)], f"rank {rank}: composites {composites}"
                if k == 2:       # one rank interrupted: it returns its input, the others blend placeholders of its outputs
                    assert got is x_r if state.interrupted else got is ex.x_out
                    d.gather_latent(ex.x_out)             # every rank still reaches the same collectives
                    continue
                assert got is ex.x_out
                for (a, b) in valid:
                    assert torch.equal(got[:, :, a:b], want[:, :, a:b]), f"rank {rank} bg={bg} step {k}: rows [{a},{b}) differ"
                full = d.gather_latent(got)
                assert torch.equal(full, want), f"rank {rank} bg={bg} step {k}: gathered latent differs"
                everyone = [None] * world
                dist.all_gather_object(everyone, list(calls))
                assert sorted(j for cl in everyone for j in cl) == list(range(len(ROWS)))
            assert ex.blends == (4 if bg else 0)
            host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_strip_shard_delegate_with_regions_equals_single(tmp_path, world):
    mp.spawn(_gloo_strip_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


def _gloo_mod_interrupt_worker(rank, world, port, result_dir):
    """Mixture of Diffusers' tile shard WITHOUT regions: an interrupted rank still joins the tile all-gather (its peers would
    wait in it forever otherwise), returns its input, and the next step is exact on every rank again."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    _install_oracle_engine()
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = c["N"]
        state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
        host.use_shared(types.SimpleNamespace(state=state, sd_model=None))
        d, step = _delegate("mod", True, True, [], rows=[])
        plan = tiling.GridPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], True)
        x = synth.latent(90, (N, c["C"], c["H"], c["W"]), torch.float16)
        want = blend.mixture_step(x, plan.batched_bboxes, plan.tile_weights, plan.rescale_factor, lambda t, bb: synth.fake_denoise(t, bb, N))
        state.interrupted = rank == world - 1
        got = step(x)
        if state.interrupted:
            assert torch.equal(got, x)
        state.interrupted = False
        assert torch.equal(step(x), want), f"rank {rank}: not in lock-step after an interrupt"
        MixtureOfDiffusers.unhook()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


def test_gloo_mixture_shard_interrupt_keeps_lock_step(tmp_path):
    mp.spawn(_gloo_mod_interrupt_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()


def test_tile_shard_needs_a_grid_or_regions():
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion
    d = MultiDiffusion(_p(GRID), _sampler())
    with pytest.raises(RuntimeError, match="init_grid_bbox"):
        d.init_tile_shard(None)


# ------------------------------------------------------------------------------------------------ GPU: the rows kernel
def _random_regions(gen, n, N, C, H, W, dt, mixture):
    regions = []
    for k in range(n):
        x0 = int(torch.randint(0, W - 1, (1,), generator=gen))
        y0 = int(torch.randint(0, H - 1, (1,), generator=gen))
        w = int(torch.randint(1, W - x0 + 1, (1,), generator=gen))
        h = int(torch.randint(1, H - y0 + 1, (1,), generator=gen))
        mode = k % 2 if k < 6 else int(torch.randint(0, 2, (1,), generator=gen))
        out = (torch.randn((N, C, h, w), generator=gen) * 1.5).to(dt)
        if mode == 1:
            aux = torch.rand((h, w), generator=gen)
        else:
            aux = torch.rand((1, 1, h, w), generator=gen) * 3 if mixture else None
        regions.append((x0, y0, w, h, mode, out.cuda(), None if aux is None else aux.cuda()))
    return regions


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("mixture", [False, True])
def test_region_composite_rows_equals_whole_canvas_rows(dn, mixture):
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel
    dt = DTYPES[dn]
    N, C, H, W, tw, th, ov = 2, 4, 200, 72, 32, 24, 8
    g = engine.make_grid(W, H, tw, th, ov, 4)
    ys = list(g.ys[:g.rows])
    gen = torch.Generator().manual_seed(5 + mixture)
    xb = (torch.randn((N, C, H, W), generator=gen) * 2).to(dt).cuda()
    weights = None if mixture else torch.randint(0, 5, (H, W), generator=gen).float().cuda()
    for n in (0, 1, 5, _cabi.TD_MAX_REGIONS):
        regions = _random_regions(gen, n, N, C, H, W, dt, mixture)
        want = engine.region_composite(xb, weights, regions)
        sentinel = torch.full((N, C, H, W), float("nan"))
        full = engine.region_composite_rows(xb, weights, regions, 0, H, sentinel.clone().cuda())
        assert_bit_equal(full.cpu(), want.cpu(), f"[0, H) {dn} n={n}")
        for world in range(2, 9):
            got = sentinel.clone().cuda()
            for r in range(world):
                lo, hi = parallel.StripShard(ys, g.cols, th, H, r, world).strip()
                one = engine.region_composite_rows(xb, weights, regions, lo, hi, sentinel.clone().cuda()).cpu()
                assert_bit_equal(one[:, :, :lo], sentinel[:, :, :lo], "rows above the window were written")
                assert_bit_equal(one[:, :, hi:], sentinel[:, :, hi:], "rows below the window were written")
                assert_bit_equal(one[:, :, lo:hi], want[:, :, lo:hi].cpu(), f"{dn} n={n} world {world} rank {r}")
                # the same regions clipped to the window: only the rows they cover there, read from row-offset views
                clipped = []
                for (x0, y0, w, h, m, o, a) in regions:
                    a0, b0 = max(y0, lo), min(y0 + h, hi)
                    if b0 > a0:
                        ac = None if a is None else a.reshape(h, w)[a0 - y0:b0 - y0]
                        clipped.append((x0, a0, w, b0 - a0, m, o[:, :, a0 - y0:b0 - y0], ac))
                engine.region_composite_rows(xb, weights, clipped, lo, hi, got)
            assert_bit_equal(got.cpu(), want.cpu(), f"{dn} n={n} world {world}: union of clipped strips")


@pytest.mark.gpu
def test_region_composite_rows_rejects_bad_windows():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine
    xb = torch.zeros((1, 4, 16, 16), device="cuda")
    out = torch.zeros_like(xb)
    for lo, hi in ((-1, 4), (5, 4), (0, 17)):
        with pytest.raises(_cabi.TdError, match="rows"):
            engine.region_composite_rows(xb, None, [], lo, hi, out)
    assert engine.region_composite_rows(xb, None, [], 8, 8, out) is out


# ------------------------------------------------------------------------------------------------ two or more GPUs
def _gpu_region_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion, MixtureOfDiffusers, host
    torch.cuda.set_device(rank)
    _init(rank, world, port, "nccl")
    try:
        c = dict(GRID, W=128, H=96)
        N = c["N"]
        host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=None))
        xs = [synth.latent(60 + k, (N, c["C"], c["H"], c["W"]), torch.float16) for k in range(3)]
        for method, mode, fused, bg in (("md", "strip", True, True), ("md", "strip", True, False), ("md", "replicate", True, True),
                                        ("md", "replicate", False, True), ("mod", "replicate", False, True), ("mod", "replicate", False, False)):
            wants = []
            for x in xs:      # the single-GPU run of the same delegate (no shard)
                d1 = (MultiDiffusion if method == "md" else MixtureOfDiffusers)(_p(c), _sampler())
                d1.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
                d1.init_custom_bbox({i: row for i, row in enumerate(ROWS)}, bg, False)
                d1.init_done()
                wants.append(_single_step(d1, method, x.cuda(), N).cpu())
            d = (MultiDiffusion if method == "md" else MixtureOfDiffusers)(_p(c), _sampler())
            d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
            d.init_custom_bbox({i: row for i, row in enumerate(ROWS)}, bg, False)
            d.init_done()
            d.init_tile_shard(None, fused=fused, mode=mode)
            for k, x in enumerate(xs):
                out = _single_step(d, method, x.cuda(), N)
                torch.cuda.synchronize()
                if mode == "strip":
                    lo, hi = d._strip.strip()
                    assert torch.equal(out[:, :, lo:hi].cpu(), wants[k][:, :, lo:hi]), f"rank {rank} {method} strip rows step {k}"
                    for (q, a, b) in d._strip.x_in():
                        assert torch.equal(out[:, :, a:b].cpu(), wants[k][:, :, a:b]), f"rank {rank}: latent halo from {q} step {k}"
                    dist.barrier()
                full = d.gather_latent(out)
                assert torch.equal(full.cpu(), wants[k]), f"rank {rank} {method} {mode} fused={fused} bg={bg} step {k}"
                dist.barrier()
            dist.barrier()
            if d._strip_exchange is not None:
                d._strip_exchange.close()
            if d._exchange is not None:
                d._exchange.close()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


def _single_step(d, method, x, N):
    def custom(x_tile, bbox_id, bbox):
        return synth.fake_region_denoise(x_tile, bbox_id)
    if method == "md":
        return d.sample_one_step(x, None, lambda t, bb: synth.fake_denoise(t, bb, N), custom)
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    batches = d.local_batched_bboxes if d._shard is not None else d.batched_bboxes
    it = {"i": 0}

    def apply_model(x_tile, t, c_):
        bb = batches[it["i"]]
        it["i"] += 1
        return synth.fake_denoise(x_tile, bb, N)
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: custom(x_tile, bbox_id, bbox)
    d.hook()
    cond = {"c_crossattn": [torch.zeros(N, 2, 4, device=x.device)], "c_concat": [torch.zeros(N, 5, 1, 1, device=x.device)]}
    out = model.apply_model(x, torch.ones(N, device=x.device), cond).clone()
    d.unhook()
    return out


@pytest.mark.gpu
def test_one_rank_shard_with_regions_bit_identical_to_unsharded(tmp_path):
    """Every shard mode with regions on a one-rank NCCL group: the real kernels and exchanges (strip blend with the
    accumulator, td_region_composite_rows into the strip's latent buffer, peer blend, all-gathers) against the unsharded
    delegate."""
    mp.spawn(_gpu_region_worker, args=(1, _free_port(), str(tmp_path)), nprocs=1, join=True)
    assert (tmp_path / "ok0").exists()


@pytest.mark.gpu
def test_multi_gpu_sharded_regions_bit_identical_to_one_gpu(tmp_path):
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs 2 GPUs")
    world = min(world, 4)
    mp.spawn(_gpu_region_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
