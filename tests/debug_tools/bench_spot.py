"""SpotDiffusion: device time per denoiser call of what runs around the UNet, against MultiDiffusion, and windows per call.

    python tests/debug_tools/bench_spot.py [--iters 2000]

fp16 latents.  Per call SpotDiffusion runs td_grid_counts (count canvas + reciprocals) + td_scatter_tiles + td_blend_multidiffusion
on its step plan (overlap 0); MultiDiffusion runs the scatter and the blend on its fixed plan, at overlap 48 (the UI default) and
at overlap 0.  Geometries: cfg2's [2,4,512,512] latent with tile 96, bounded and wrapped in x and y, and the [2,4,512,2048]
panorama wrapped in x.  Times are CUDA events around replays of a CUDA graph of 20 calls (bench_wrap.time_us); the step
plan is the one of the first draw of seed 0, whose window count is that of every call.  The UNet time is not part of this:
its saving is the window count.  Prints the card name and power limit read in the same run.
"""
import argparse
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_wrap import card, time_us  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import engine  # noqa: E402

TILE, BS = 96, 4


def _tile_outs(g, x, N):
    tiles = engine.scatter_tiles(g, x)
    return tiles, [tiles[b * g.tile_bs * N:min((b + 1) * g.tile_bs, g.num_tiles) * N].clone() for b in range(g.num_batches)]


def multidiffusion(x, overlap, wrap, iters):
    N, C, H, W = x.shape
    g = engine.make_grid(W, H, TILE, TILE, overlap, BS, wrap=wrap)
    tiles, outs = _tile_outs(g, x, N)
    w_host = engine.grid_weights(g)
    wts = torch.from_numpy(w_host).cuda()
    rcp = engine.exact_reciprocals(w_host)
    rcp = torch.from_numpy(rcp).cuda() if rcp is not None else None
    out = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")

    def call():
        engine.scatter_tiles(g, x, out=tiles)
        engine.blend_multidiffusion(g, outs, N, C, g.tile_bs, wts, x.dtype, out=out, rcp_weights=rcp)
    return dict(method=f"MultiDiffusion overlap {overlap}", windows=g.num_tiles, us=round(time_us(call, iters), 2))


def spotdiffusion(x, wrap, iters):
    N, C, H, W = x.shape
    base = engine.make_grid(W, H, TILE, TILE, 0, BS, wrap=wrap)
    lo_x, hi_x, lo_y, hi_y = engine.shift_bounds(base)
    rng = random.Random(0)
    sx = rng.randrange(lo_x, hi_x) if hi_x - lo_x > 1 else lo_x
    sy = rng.randrange(lo_y, hi_y) if hi_y - lo_y > 1 else lo_y
    g = engine.shift_grid(base, sx, sy, BS)
    tiles, outs = _tile_outs(g, x, N)
    wts = torch.empty((H, W), dtype=torch.float32, device="cuda")
    rcp = torch.empty((H, W), dtype=torch.float32, device="cuda") if engine.counts_allow_fast_divide(g) else None
    out = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")

    def counts():
        engine.grid_counts(g, wts, rcp)

    def call():
        engine.grid_counts(g, wts, rcp)
        engine.scatter_tiles(g, x, out=tiles)
        engine.blend_multidiffusion(g, outs, N, C, g.tile_bs, wts, x.dtype, out=out, rcp_weights=rcp)
    counts_us = time_us(counts, iters)
    return dict(method="SpotDiffusion overlap 0", windows=g.num_tiles, us=round(time_us(call, iters), 2), counts_us=round(counts_us, 2),
                counts_mbytes=round(H * W * (8 if rcp is not None else 4) / 1e6, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_spot measures on the GPU"
    print(json.dumps({"card": card()}))
    shapes = [("cfg2 [2,4,512,512] bounded", (2, 4, 512, 512), 0),
              ("cfg2 [2,4,512,512] wrap xy", (2, 4, 512, 512), engine.WRAP_X | engine.WRAP_Y),
              ("panorama [2,4,512,2048] wrap x", (2, 4, 512, 2048), engine.WRAP_X)]
    for name, shape, wrap in shapes:
        x = torch.randn(shape, device="cuda").half()
        for row in (multidiffusion(x, 48, wrap, args.iters), multidiffusion(x, 0, wrap, args.iters), spotdiffusion(x, wrap, args.iters)):
            print(json.dumps(dict(shape=name, **row)))


if __name__ == "__main__":
    main()
