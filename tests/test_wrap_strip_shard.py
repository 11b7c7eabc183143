"""MultiDiffusion and Mixture of Diffusers under the row-strip tile shard on a wrapped grid (seamless tiling), on CPU.

The delegates' strip tails run on gloo processes (2 and 3 ranks) with the device kernels swapped for tests/wrap_oracle.py and an
exchange stand-in that blends each rank's own rows with the wrap oracle; each rank's input is valid only on its strip and its
latent halo, which under wrap_y includes rows from the top of the canvas.  Own rows, halo rows and the gathered latent must
equal the unsharded wrapped delegate (on the same oracle engine) every step, grid only and with BACKGROUND / FOREGROUND
regions.  init_tile_shard() without an explicit mode still refuses a wrapped grid."""
import os
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import wrap_oracle as wo
from helpers import region_composite_reference
from oracle import synth
from test_region_shard import ROWS, _BG, _free_port, _init, _p, _sampler

GRID = dict(N=2, C=4, W=64, H=48, tw=16, th=16, ov=8, bs=4)
XY = wo.WRAP_X | wo.WRAP_Y


def _install_wrap_oracle_engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200.tile_methods import abstractdiffusion

    def bbs(g):
        return [tuple(int(v) for v in r) for r in engine.grid_bboxes_xywh(g)]

    def scatter_tiles(g, x, out=None, tile_begin=0, tile_end=None, flags=0):
        return wo.scatter(x, bbs(g)[tile_begin:tile_end])

    def blend_multidiffusion(g, outs, N, C, tile_bs, weights, acc_dtype, x_buffer=None, flags=0, out=None, rcp_weights=None):
        buf = torch.zeros((N, C, g.H, g.W), dtype=acc_dtype)
        wo.accumulate_md(buf, torch.cat(list(outs), dim=0), bbs(g), N)
        if x_buffer is not None:
            x_buffer.copy_(buf)
        return wo.normalise_md(buf, weights.to(buf.device))

    def blend_mixture(g, outs, N, C, tile_bs, tile_weights, rescale, x_buffer, flags=0):
        x_buffer.zero_()
        wo.accumulate_mod(x_buffer, torch.cat(list(outs), dim=0), bbs(g), N, tile_weights.to(x_buffer.device), rescale.to(x_buffer.device))
        return x_buffer

    def region_composite_rows(x_buffer, weights, regions, row_begin, row_end, out):
        out[:, :, row_begin:row_end] = region_composite_reference(x_buffer, weights, regions)[:, :, row_begin:row_end]
        return out

    engine.scatter_tiles, engine.blend_multidiffusion, engine.blend_mixture = scatter_tiles, blend_multidiffusion, blend_mixture
    engine.region_composite, engine.region_composite_rows = region_composite_reference, region_composite_rows
    abstractdiffusion.AbstractDiffusion._check_input = lambda self, x: x.contiguous()


class _WrapOracleStripExchange:
    """parallel.StripExchange's interface on CPU tensors over gloo: the tile outputs of all ranks are all-gathered and the wrap
    oracle blends the OWN rows only; the latent halo (rows at their canvas position, from the top of the canvas too under
    wrap_y) and `gather_latent` move strips with all-gathers.  Rows a rank neither owns nor receives stay NaN."""

    def __init__(self, d, N, C, dtype, latent_dtype):
        self.d, self.sh, self.N, self.C, self.dtype = d, d._strip, N, C, dtype
        self.x_out = torch.full((N, C, d.h, d.w), float("nan"), dtype=latent_dtype)
        self.blends = 0

    def own_tiles(self):
        t0, t1 = self.sh.tile_range()
        self._own = torch.empty(((t1 - t0) * self.N, self.C, self.sh.tile_h, self.d.tile_w), dtype=self.dtype)
        return self._own

    def push_tile_halos(self):
        pass

    def _all_tiles(self):
        sh, N = self.sh, self.N
        most = max(sh.tile_range(r)[1] - sh.tile_range(r)[0] for r in range(sh.world)) * N
        pad = torch.zeros((most,) + tuple(self._own.shape[1:]), dtype=self.dtype)
        pad[:self._own.shape[0]] = self._own
        parts = [torch.empty_like(pad) for _ in range(sh.world)]
        dist.all_gather(parts, pad)
        return torch.cat([parts[r][:(sh.tile_range(r)[1] - sh.tile_range(r)[0]) * N] for r in range(sh.world)])

    def blend(self, g, weights, rcp_weights, flags=0, x_buffer=None):
        from multidiffusion_upscaler_for_automatic1111_b200 import engine
        acc = torch.zeros((self.N, self.C, g.H, g.W), dtype=self.dtype)
        wo.accumulate_md(acc, self._all_tiles(), [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)], self.N)
        lo, hi = self.sh.strip()
        self.x_out[:, :, lo:hi] = wo.normalise_md(acc, weights.cpu())[:, :, lo:hi]
        if x_buffer is not None:
            x_buffer[:, :, lo:hi] = acc[:, :, lo:hi]
        self.blends += 1
        return self.x_out

    def blend_mixture(self, g, tile_weights, rescale, flags=0, x_buffer=None):
        from multidiffusion_upscaler_for_automatic1111_b200 import engine
        acc = torch.zeros((self.N, self.C, g.H, g.W), dtype=self.dtype)
        wo.accumulate_mod(acc, self._all_tiles(), [tuple(int(v) for v in b) for b in engine.grid_bboxes_xywh(g)], self.N, tile_weights.cpu(),
                          rescale.cpu())
        out = x_buffer if x_buffer is not None else self.x_out
        lo, hi = self.sh.strip()
        out[:, :, lo:hi] = acc[:, :, lo:hi]
        self.blends += 1
        return out

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


def _make(method, wrap, rows):
    """A delegate on the wrapped GRID with `rows` (may be empty) and its one-step function."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    c = GRID
    N = c["N"]
    d = (MultiDiffusion if method == "md" else MixtureOfDiffusers)(_p(c), _sampler())
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"], wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    if rows:
        d.init_custom_bbox({i: row for i, row in enumerate(rows)}, True, False)
    d.init_done()
    if method == "md":
        return d, lambda x: d.sample_one_step(x, None, lambda t, bb: synth.fake_denoise(t, bb, N),
                                              lambda xt, j, bb: synth.fake_region_denoise(xt, j))

    def step(x):
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
        try:
            return model.apply_model(x, torch.ones(N), {"c_crossattn": [torch.zeros(N, 2, 4)], "c_concat": [torch.zeros(N, 5, 1, 1)]})
        finally:
            d.unhook()
    return d, step


SCENARIOS = {"grid only": [], "background regions": [r for r in ROWS if r[7] == _BG], "foreground regions": ROWS}


def _gloo_wrap_strip_worker(rank, world, port, result_dir):
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    _install_wrap_oracle_engine()
    _init(rank, world, port, "gloo")
    try:
        c = GRID
        N = c["N"]
        host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=None))
        for method in ("md", "mod"):
            for wrap in (wo.WRAP_X, XY):
                for name, rows in SCENARIOS.items():
                    what = f"rank {rank} {method} wrap {wrap} {name}"
                    xs = [synth.latent(150 + k, (N, c["C"], c["H"], c["W"]), torch.float16) for k in range(3)]
                    ref, ref_step = _make(method, wrap, rows)
                    wants = [ref_step(x).clone() for x in xs]
                    d, step = _make(method, wrap, rows)
                    with pytest.raises(NotImplementedError, match="explicit"):
                        d.init_tile_shard(None)
                    d.init_tile_shard(None, fused=True, mode="strip")
                    sh = d._strip
                    assert d._shard_mode == "strip" and sh.wrap_y == bool(wrap & wo.WRAP_Y)
                    d._strip_exchange = ex = _WrapOracleStripExchange(d, N, c["C"], torch.float16, d._strip_latent_dtype(torch.float16))
                    lo, hi = sh.strip()
                    valid = [(lo, hi)] + [(a, b) for (_, a, b) in sh.x_in()]
                    if wrap & wo.WRAP_Y and rank == world - 1:
                        assert any(a == 0 for (_, a, b) in sh.x_in()), f"{what}: the last strip must read rows from the top"
                    for k, x in enumerate(xs):
                        x_r = torch.full_like(x, float("nan"))
                        for (a, b) in valid:
                            x_r[:, :, a:b] = x[:, :, a:b]
                        got = step(x_r)
                        assert got is ex.x_out and got.dtype == wants[k].dtype, f"{what} step {k}"
                        for (a, b) in valid:
                            assert torch.equal(got[:, :, a:b], wants[k][:, :, a:b]), f"{what} step {k}: rows [{a},{b}) differ"
                        full = d.gather_latent(got)
                        assert torch.equal(full, wants[k]), f"{what} step {k}: gathered latent differs"
                    assert ex.blends == 3
                    dist.barrier()
        host.use_shared(None)
        open(os.path.join(result_dir, f"ok{rank}"), "w").close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_wrapped_strip_delegates_equal_single(tmp_path, world):
    mp.spawn(_gloo_wrap_strip_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
