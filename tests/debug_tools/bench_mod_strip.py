"""Mixture of Diffusers under the row-strip tile shard: kernel times of the row-window gaussian blend, and (two or more GPUs)
the delegate's step in replicate and in strip mode.

    python tests/debug_tools/bench_mod_strip.py [--iters 2000] [--baseline-lib OTHER/libtd_b200.so]
    torchrun --nproc-per-node K tests/debug_tools/bench_mod_strip.py --steps 50

One GPU, BASELINE cfg3's geometry (latent [2,4,512,512] fp16, tile 96, overlap 48, tile_bs 4: 10 x 10 tiles): td_blend_mixture
over the whole canvas, and td_blend_mixture_rows for every strip of worlds 2, 4 and 8, without a wait and with a wait on flags
that are already satisfied (the production own-band setting).  Each timed call reads the next of --buffer-sets cold copies
of the tile outputs and writes the next latent (as bench.py rotates its buffers), 20 calls per CUDA graph, CUDA events around
the replays.  With --baseline-lib the same whole-canvas call of another build of the library (e.g. the parent commit's) is
timed in the same process, alternating with this build's.  The card's name and power limit are read in the same run.

Under torchrun with K >= 2 ranks: the MixtureOfDiffusers delegate (identity denoiser) in replicate and in strip mode, ms per
step (host clock around --steps steps ending in a device synchronise), the bytes a rank moves per step computed from the plan,
and an in-run check that the gathered strip latent is bit-equal to the replicate result.  On one GPU this part is skipped.
"""
import argparse
import ctypes
import json
import os
import sys
import time
import types

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_wrap import card  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, parallel  # noqa: E402

CFG3 = dict(N=2, C=4, H=512, W=512, tile=96, overlap=48, tile_bs=4)


def time_graph_us(calls, iters, per_graph=20):
    """Per-call time of `calls` (a list of closures, used round-robin): per_graph calls captured in one CUDA graph, replayed,
    timed with events."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for fn in calls[:3]:
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(per_graph):
            calls[i % len(calls)]()
    reps = max(1, iters // per_graph)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * per_graph)


def _baseline_blend(path):
    lib = ctypes.CDLL(path)
    fn = lib.td_blend_mixture
    fn.restype = ctypes.c_int
    fn.argtypes = _cabi._SIGNATURES["td_blend_mixture"][1]
    return fn


def one_gpu(args):
    from oracle import tiling
    c = CFG3
    N, C, H, W, dt = c["N"], c["C"], c["H"], c["W"], torch.float16
    g = engine.make_grid(W, H, c["tile"], c["tile"], c["overlap"], c["tile_bs"])
    tw_host = tiling.gaussian_weights(g.tile_w, g.tile_h)
    tw_d = torch.from_numpy(tw_host).cuda()
    rs_d = torch.from_numpy(engine.rescale_factor(engine.grid_weights(g, tw_host))).cuda()
    x = torch.randn((N, C, H, W), device="cuda").to(dt)
    K = args.buffer_sets
    tiles = [engine.scatter_tiles(g, x).mul_(1 + 0.01 * k) for k in range(K)]
    outs = [torch.empty_like(x) for _ in range(K)]
    batches = [[t[b * g.tile_bs * N:min((b + 1) * g.tile_bs, g.num_tiles) * N] for b in range(g.num_batches)] for t in tiles]
    band = g.cols * N * C * g.tile_h * g.tile_w * 2
    rows_ptrs = [[t.data_ptr() + i * band for i in range(g.rows)] for t in tiles]
    res = {"card": card(), "geometry": f"latent [{N},{C},{H},{W}] fp16, tile {c['tile']}, overlap {c['overlap']}, {g.rows} x {g.cols} tiles",
           "buffer_sets": K}

    def whole(k, fn=None):
        if fn is None:
            return lambda: engine.blend_mixture(g, batches[k], N, C, g.tile_bs, tw_d, rs_d, outs[k])
        ptrs = (ctypes.c_void_p * g.num_batches)(*[b.data_ptr() for b in batches[k]])
        code = _cabi.dtype_code(dt)
        return lambda: _cabi.check(fn(ctypes.byref(g), ptrs, g.num_batches, g.tile_bs, N, C, code, code, tw_d.data_ptr(), rs_d.data_ptr(),
                                      outs[k].data_ptr(), 0, _cabi.current_stream_ptr()))

    # whole canvas: this build, and (alternating, same process) the baseline build
    base = _baseline_blend(args.baseline_lib) if args.baseline_lib else None
    if base is not None:
        ref = torch.empty_like(x)
        engine.blend_mixture(g, batches[0], N, C, g.tile_bs, tw_d, rs_d, ref)
        whole(0, base)()
        torch.cuda.synchronize()
        res["baseline_bit_equal"] = bool(torch.equal(ref.view(torch.int16), outs[0].view(torch.int16)))
    t_this, t_base = [], []
    for _ in range(args.rounds):
        t_this.append(time_graph_us([whole(k) for k in range(K)], args.iters))
        if base is not None:
            t_base.append(time_graph_us([whole(k, base) for k in range(K)], args.iters))
    res["whole_canvas_us"] = {"this": [round(v, 2) for v in t_this]}
    if base is not None:
        res["whole_canvas_us"]["baseline"] = [round(v, 2) for v in t_base]
    # one strip per rank of worlds 2, 4, 8; no wait, and a wait on flags already satisfied (own bands as production)
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    flags[:32] = 7
    flags[32] = 7
    ys = list(g.ys[:g.rows])
    for world in (2, 4, 8):
        per = []
        for r in range(world):
            sh = parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world)
            lo, hi = sh.strip()
            first, count = sh.wait_range("tiles")
            row = {"rank": r, "rows": [lo, hi]}
            for label, wait in (("no_wait", None), ("wait_satisfied", (ctypes.c_void_p(flags.data_ptr() + 4 * first), max(count, 1),
                                                                          ctypes.c_void_p(flags.data_ptr() + 128)))):
                def call(k, wait=wait, lo=lo, hi=hi, sh=sh):
                    return lambda: engine.blend_mixture_rows(g, rows_ptrs[k], N, C, dt, tw_d, rs_d, outs[k], lo, hi, wait=wait,
                                                             own_bands=(sh.band_begin[r], sh.band_end[r]))
                row[label + "_us"] = round(time_graph_us([call(k) for k in range(K)], args.iters), 2)
            per.append(row)
        res[f"world_{world}"] = {"strips": per, "slowest_strip_us": {k: max(p[k] for p in per) for k in ("no_wait_us", "wait_satisfied_us")}}
    torch.cuda.synchronize()
    assert flags[:33].tolist() == [7] * 33, "a timed launch moved the flags"
    return res


def plan_bytes(d, N, C, es):
    """Bytes a rank sends per step: replicate = its padded chunk of the tile all-gather (every rank receives world x that);
    strip = the tile-halo rows it pushes + the latent-halo rows it pushes."""
    g = d._grid
    tile = N * C * g.tile_h * g.tile_w * es
    if d._strip is None:
        return {"tile_all_gather_send": d._shard.chunk * tile, "tile_all_gather_receive": d._shard.chunk * tile * (d._shard.world - 1)}
    sh = d._strip
    tiles = sum((v1 - v0) * g.tile_w * g.cols * N * C * es for (_, _, v0, v1) in sh.halo_out())
    lat = sum((b - a) * g.W * N * C * es for (_, a, b) in sh.x_out())
    return {"tile_halo_send": tiles, "latent_halo_send": lat}


def multi_gpu(args):
    import torch.distributed as dist
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, host
    rank, world = dist.get_rank(), dist.get_world_size()
    c = CFG3
    N, C, H, W, dt = c["N"], c["C"], c["H"], c["W"], torch.float16
    host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=None))
    x = torch.randn((N, C, H, W), generator=torch.Generator().manual_seed(1)).to(dt).cuda()
    res = {}
    latents = {}
    for mode in ("replicate", "strip"):
        d = MixtureOfDiffusers(types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a", disable_extra_networks=True),
                               types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None),
                                                                                          image_cfg_scale=None, step=0)))
        d.init_grid_bbox(c["tile"], c["tile"], c["overlap"], c["tile_bs"])
        d.init_done()
        d.init_tile_shard(None, fused=True, mode=mode)
        model = types.SimpleNamespace(apply_model=lambda x_tile, t, c_: x_tile, cond_stage_key="txt",
                                      model=types.SimpleNamespace(conditioning_key="crossattn"))
        host.get_shared().sd_model = model
        d.hook()
        cond = {"c_crossattn": [torch.zeros(N, 2, 4, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
        for _ in range(3):
            out = model.apply_model(x, torch.ones(N, device="cuda"), cond)
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            out = model.apply_model(x, torch.ones(N, device="cuda"), cond)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / args.steps
        latents[mode] = d.gather_latent(out).clone()
        res[mode] = {"ms_per_step": round(ms, 3), "bytes_per_step": plan_bytes(d, N, C, 2)}
        d.unhook()
        if d._strip_exchange is not None:
            d._strip_exchange.close()
    res["strip_bit_equal_to_replicate"] = bool(torch.equal(latents["strip"].view(torch.int16), latents["replicate"].view(torch.int16)))
    assert res["strip_bit_equal_to_replicate"], "the gathered strip latent differs from the replicate result"
    return rank, world, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of this build's and the baseline's whole-canvas timing")
    ap.add_argument("--buffer-sets", type=int, default=8)
    ap.add_argument("--baseline-lib", default=None, help="another build of libtd_b200.so whose td_blend_mixture is timed alongside")
    ap.add_argument("--steps", type=int, default=50, help="multi-GPU part: timed delegate steps per mode")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mod_strip measures on the GPU"
    if int(os.environ.get("WORLD_SIZE", "1")) >= 2:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
        try:
            rank, world, res = multi_gpu(args)
            if rank == 0:
                print(json.dumps({"multi_gpu": {"world": world, "card": card(), **res}}))
        finally:
            dist.destroy_process_group()
        return
    print(json.dumps({"one_gpu": one_gpu(args)}))
    print(json.dumps({"multi_gpu": f"skipped: {torch.cuda.device_count()} GPU(s) visible, run under torchrun with >= 2 ranks"}))


if __name__ == "__main__":
    main()
