"""Mixture of Diffusers under the row-strip tile shard (init_tile_shard(mode="strip")), on CPU.

The delegate's strip tail (`apply_model_hijack` -> `_apply_strip` -> `_strip_step`) runs on gloo processes with the device
kernels swapped for the oracle and an exchange stand-in that blends with `oracle.blend.accumulate_mod`; each rank's input is
valid only on its strip and latent halo.  Own rows, halo rows and the gathered latent must equal the single-process oracle
every step, with and without regions, and after an interrupt on one rank.  Also: the default shard mode stays "replicate",
and the refusals (latent width, a change of N or dtype, noise inversion)."""
import os
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import region_composite_reference
from oracle import blend, synth, tiling
from test_region_shard import GRID, ROWS, _BG, _OracleStripExchange, _free_port, _init, _install_oracle_engine, _oracle_step, _p, _sampler


class _OracleMixtureStripExchange(_OracleStripExchange):
    """_OracleStripExchange with the Mixture-of-Diffusers blend: the latent buffer has the latent dtype (fp32 with FOREGROUND
    regions), and the strip rows are blended with accumulate_mod into it, or into x_buffer when regions follow."""

    def __init__(self, d, N, C, dtype, latent_dtype):
        super().__init__(d, N, C, dtype)
        self.x_out = self.x_out.to(latent_dtype)

    def blend(self, *args, **kwargs):
        raise AssertionError("Mixture of Diffusers must not run the MultiDiffusion blend")

    def blend_mixture(self, g, tile_weights, rescale, flags=0, x_buffer=None):
        from multidiffusion_upscaler_for_automatic1111_b200 import engine
        sh, N = self.sh, self.N
        most = max(sh.tile_range(r)[1] - sh.tile_range(r)[0] for r in range(sh.world)) * N
        pad = torch.zeros((most,) + tuple(self._own.shape[1:]), dtype=self.dtype)
        pad[:self._own.shape[0]] = self._own
        parts = [torch.empty_like(pad) for _ in range(sh.world)]
        dist.all_gather(parts, pad)
        tiles = torch.cat([parts[r][:(sh.tile_range(r)[1] - sh.tile_range(r)[0]) * N] for r in range(sh.world)])
        acc = torch.zeros((N, self.C, g.H, g.W), dtype=self.dtype)
        blend.accumulate_mod(acc, tiles, [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)], N, tile_weights.cpu(), rescale.cpu())
        out = x_buffer if x_buffer is not None else self.x_out
        lo, hi = sh.strip()
        out[:, :, lo:hi] = acc[:, :, lo:hi]
        self.blends += 1
        return out


def _mod_delegate(rows, bg, mode="strip"):
    """A MixtureOfDiffusers delegate on GRID with `rows` (may be empty), sharded in `mode`; returns (delegate, step(x))."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, host
    c = GRID
    N = c["N"]
    d = MixtureOfDiffusers(_p(c), _sampler())
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"])
    if rows:
        d.init_custom_bbox({i: row for i, row in enumerate(rows)}, bg, False)
    d.init_done()
    d.init_tile_shard(None, fused=True, mode=mode)
    it = {"i": 0}

    def apply_model(x_tile, t, c_):
        bb = d.local_batched_bboxes[it["i"]]
        it["i"] += 1
        return synth.fake_denoise(x_tile, bb, x_tile.shape[0] // len(bb))
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    d.custom_apply_model = lambda x_tile, t, c_, bbox_id, bbox: synth.fake_region_denoise(x_tile, bbox_id)
    d.hook()

    def step(x):
        it["i"] = 0
        n = x.shape[0]
        return model.apply_model(x, torch.ones(n), {"c_crossattn": [torch.zeros(n, 2, 4)], "c_concat": [torch.zeros(n, 5, 1, 1)]})
    return d, step


def _want(x, rows, bg):
    c = GRID
    N = x.shape[0]
    if not rows:
        plan = tiling.GridPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], True)
        return blend.mixture_step(x, plan.batched_bboxes, plan.tile_weights, plan.rescale_factor, lambda t, bb: synth.fake_denoise(t, bb, N))
    return _oracle_step("mod", x, bg, rows)


SCENARIOS = {"grid only": ([], True), "background regions": ([r for r in ROWS if r[7] == _BG], True),
             "foreground regions": (ROWS, True), "no background layer": (ROWS, False)}


def _gloo_mod_strip_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, engine, host
    _install_oracle_engine()
    composites = []

    def region_composite_rows(x_buffer, weights, regions, row_begin, row_end, out):
        assert out.dtype == torch.float32 and tuple(out.shape) == tuple(x_buffer.shape)
        composites.append((row_begin, row_end))
        out[:, :, row_begin:row_end] = region_composite_reference(x_buffer, weights, regions)[:, :, row_begin:row_end]
        return out
    engine.region_composite_rows = region_composite_rows
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = c["N"]
        state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
        host.use_shared(types.SimpleNamespace(state=state, sd_model=None))
        d, _ = _mod_delegate([], True, mode=None)
        assert d._shard_mode == "replicate", "the default shard mode of Mixture of Diffusers must stay replicate"
        MixtureOfDiffusers.unhook()
        for name, (rows, bg) in SCENARIOS.items():
            d, step = _mod_delegate(rows, bg)
            assert d._shard_mode == "strip" and d._strip is not None
            sh = d._strip
            fg = any(r[7] != _BG for r in rows)
            d._strip_exchange = ex = _OracleMixtureStripExchange(d, N, c["C"], torch.float16, d._strip_latent_dtype(torch.float16))
            assert ex.x_out.dtype == (torch.float32 if fg else torch.float16)
            lo, hi = sh.strip()
            valid = [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]
            for k in range(4):
                x = synth.latent(120 + k, (N, c["C"], c["H"], c["W"]), torch.float16)
                want = _want(x, rows, bg)
                x_r = torch.full_like(x, float("nan"))        # what this rank holds: its strip and latent halo
                for (a, b) in valid:
                    x_r[:, :, a:b] = x[:, :, a:b]
                state.interrupted = k == 2 and rank == world - 1
                del composites[:]
                got = step(x_r)
                assert composites == ([(lo, hi)] if rows else []), f"rank {rank} {name}: composites {composites}"
                if k == 2:       # one rank interrupted: it returns its input, the others blend placeholders of its outputs
                    # (Mixture of Diffusers polls the interrupt between grid batches only: without a background layer it never sees it)
                    assert got is (x_r if state.interrupted and bg else ex.x_out), f"rank {rank} {name}: interrupted step"
                    d.gather_latent(ex.x_out)             # every rank still reaches the same collectives
                    continue
                assert got is ex.x_out and got.dtype == want.dtype, f"rank {rank} {name}: returned {got.dtype}, want {want.dtype}"
                for (a, b) in valid:
                    assert torch.equal(got[:, :, a:b], want[:, :, a:b]), f"rank {rank} {name} step {k}: rows [{a},{b}) differ"
                full = d.gather_latent(got)
                assert torch.equal(full, want), f"rank {rank} {name} step {k}: gathered latent differs"
            assert ex.blends == (4 if bg else 0)
            if not rows:
                # the exchange is built for one N and dtype: anything else is refused, not blended into a wrong latent
                with pytest.raises(ValueError, match="built for N=2"):
                    step(synth.latent(1, (N, c["C"], c["H"], c["W"]), torch.float32))
                with pytest.raises(ValueError, match="built for N=2"):
                    step(synth.latent(1, (1, c["C"], c["H"], c["W"]), torch.float16))
                # noise inversion evaluates the same hijack: refused in strip mode
                with pytest.raises(NotImplementedError, match="noise inversion"):
                    d.get_noise(x, torch.ones(N), {"c_crossattn": [torch.zeros(N, 2, 4)], "c_concat": [torch.zeros(N, 5, 1, 1)]}, 1)
            MixtureOfDiffusers.unhook()
            dist.barrier()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_mixture_strip_delegate_equals_single(tmp_path, world):
    mp.spawn(_gloo_mod_strip_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


def test_strip_mode_refuses_noise_inversion():
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers
    d = MixtureOfDiffusers(_p(GRID), _sampler())
    d.init_grid_bbox(GRID["tw"], GRID["th"], GRID["ov"], GRID["bs"])
    d.init_done()
    d.noise_inverse_enabled = True
    with pytest.raises(NotImplementedError, match="noise inversion"):
        d.init_tile_shard(None, mode="strip")


@pytest.mark.parametrize("W,dtype", [(60, torch.float16), (60, torch.bfloat16), (62, torch.float32)])
def test_exchange_refuses_latent_rows_that_are_not_16_byte_multiples(W, dtype):
    """The latent-halo rows are pushed as 16-byte vectors: W % 8 for fp16 / bf16 latents, W % 4 for fp32.  The refusal comes
    before anything is allocated or exchanged (this machine has no GPU: reaching the allocation would raise a CUDA error)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import parallel
    sh = parallel.StripShard([0, 8, 16], 1, 16, 32, 0, 1)
    with pytest.raises(ValueError, match=f"W % {16 // torch.empty((), dtype=dtype).element_size()} == 0"):
        parallel.StripExchange(sh, 1, 4, 16, W, torch.float16, torch.device("cpu"), latent_dtype=dtype)
