"""Seamless tiling under the row-strip tile shard: kernel times of the row-window wrap blends (td_blend_multidiffusion_wrap_rows,
td_blend_mixture_wrap_rows) next to the whole-canvas wrap blends on the same plan.

    python tests/debug_tools/bench_wrap_strip.py [--iters 2000] [--rounds 3]

Geometries: cfg2 wrapped in x and y (latent [2,4,512,512] fp16, tile 96, overlap 48) and the panorama wrapped in x
([2,4,512,2048]).  For MultiDiffusion and Mixture of Diffusers: the whole-canvas td_blend_*; the rows entry with window [0, H)
and no wait; and the rows entry for every strip of worlds 2, 4 and 8, without a wait and with a wait on flags that are
already satisfied (the production own-band setting).  The whole-canvas timing alternates with the others, --rounds times.
Each timed call reads the next of --buffer-sets cold copies of the tile outputs and writes the next latent, 20 calls per CUDA
graph, CUDA events around the replays.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_mod_strip import time_graph_us  # noqa: E402
from bench_wrap import card  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import engine, parallel  # noqa: E402

GEOMS = {"cfg2 xy": dict(N=2, C=4, H=512, W=512, tile=96, overlap=48, wrap=engine.WRAP_X | engine.WRAP_Y),
         "panorama x": dict(N=2, C=4, H=512, W=2048, tile=96, overlap=48, wrap=engine.WRAP_X)}


def run_geometry(name, args):
    from oracle import tiling
    c = GEOMS[name]
    N, C, H, W, dt = c["N"], c["C"], c["H"], c["W"], torch.float16
    g = engine.make_grid(W, H, c["tile"], c["tile"], c["overlap"], 4, wrap=c["wrap"])
    tw_host = tiling.gaussian_weights(g.tile_w, g.tile_h)
    tw_d = torch.from_numpy(tw_host).cuda()
    rs_d = torch.from_numpy(engine.rescale_factor(engine.grid_weights(g, tw_host))).cuda()
    wts = torch.from_numpy(engine.grid_weights(g)).cuda()
    x = torch.randn((N, C, H, W), device="cuda").to(dt)
    K = args.buffer_sets
    tiles = [engine.scatter_tiles(g, x).mul_(1 + 0.01 * k) for k in range(K)]
    outs16 = [torch.empty_like(x) for _ in range(K)]
    outs32 = [torch.empty((N, C, H, W), dtype=torch.float32, device="cuda") for _ in range(K)]
    batches = [[t[b * g.tile_bs * N:min((b + 1) * g.tile_bs, g.num_tiles) * N] for b in range(g.num_batches)] for t in tiles]
    band = g.cols * N * C * g.tile_h * g.tile_w * 2
    rows_ptrs = [[t.data_ptr() + i * band for i in range(g.rows)] for t in tiles]
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    flags[:33] = 7
    res = {"geometry": f"latent [{N},{C},{H},{W}] fp16, tile {c['tile']}, overlap {c['overlap']}, wrap {c['wrap']}, {g.rows} x {g.cols} tiles"}

    def whole(method, k):
        if method == "md":
            return lambda: engine.blend_multidiffusion(g, batches[k], N, C, g.tile_bs, wts, dt, out=outs32[k])
        return lambda: engine.blend_mixture(g, batches[k], N, C, g.tile_bs, tw_d, rs_d, outs16[k])

    def rows(method, k, lo, hi, wait=None, own=(0, 0)):
        if method == "md":
            return lambda: engine.blend_multidiffusion_wrap_rows(g, rows_ptrs[k], N, C, dt, wts, outs32[k], lo, hi, wait=wait, own_bands=own)
        return lambda: engine.blend_mixture_wrap_rows(g, rows_ptrs[k], N, C, dt, tw_d, rs_d, outs16[k], lo, hi, wait=wait, own_bands=own)

    ys = list(g.ys[:g.rows])
    for method in ("md", "mod"):
        m = {"whole_canvas_us": [], "rows_0_H_no_wait_us": []}
        for _ in range(args.rounds):        # alternated: whole canvas, then the [0, H) window
            m["whole_canvas_us"].append(round(time_graph_us([whole(method, k) for k in range(K)], args.iters), 2))
            m["rows_0_H_no_wait_us"].append(round(time_graph_us([rows(method, k, 0, H) for k in range(K)], args.iters), 2))
        for world in (2, 4, 8):
            per = []
            for r in range(world):
                sh = parallel.StripShard(ys, g.cols, g.tile_h, g.H, r, world, wrap_y=bool(g.wrap & engine.WRAP_Y))
                lo, hi = sh.strip()
                first, count = sh.wait_range("tiles")
                own = (sh.band_begin[r], sh.band_end[r])
                wait = (ctypes.c_void_p(flags.data_ptr() + 4 * first), max(count, 1), ctypes.c_void_p(flags.data_ptr() + 128))
                row = {"rank": r, "rows": [lo, hi]}
                if hi > lo:
                    row["no_wait_us"] = round(time_graph_us([rows(method, k, lo, hi) for k in range(K)], args.iters), 2)
                    row["wait_satisfied_us"] = round(time_graph_us([rows(method, k, lo, hi, wait, own) for k in range(K)], args.iters), 2)
                per.append(row)
            timed = [p for p in per if "no_wait_us" in p]
            m[f"world_{world}"] = {"strips": per, "slowest_strip_us": {k: max(p[k] for p in timed) for k in ("no_wait_us", "wait_satisfied_us")}}
            m["whole_canvas_us"].append(round(time_graph_us([whole(method, k) for k in range(K)], args.iters), 2))
        res[method] = m
    torch.cuda.synchronize()
    assert flags[:33].tolist() == [7] * 33, "a timed launch moved the flags"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--buffer-sets", type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wrap_strip measures on the GPU"
    out = {"card": card()}
    for name in GEOMS:
        out[name] = run_geometry(name, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
