"""Inpainting (init_inpaint_mask): device time of the dense blend against the sparse blend at 10%, 50% and 100% active tiles, and
the UNet evaluations an inpaint mask saves.

    python tests/debug_tools/bench_inpaint_mask.py [--iters 2000]

fp16 [2, 4, H, W] latents, tile 96, overlap 48, tile_bs 8, on cfg2's 512^2 latent (100 tiles) and on a 1024^2 latent.  The
dense blend (td_blend_multidiffusion / td_blend_mixture) blends every tile; the sparse one (td_blend_*_sparse) blends the
compact batches of the active tiles, drawn at random with a fixed seed.  Times are CUDA events around replays of a CUDA graph of
20 calls (bench_wrap.time_us).  The UNet evaluations saved are a count from the plan, not a time: the UNet calls (tile batches) of
one denoiser call with and without the mask, for a mask that reaches a 128^2 latent square in the middle of the canvas.  Prints
the card name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_wrap import card, time_us  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import engine  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import gaussian_weights  # noqa: E402

N, C, TILE, OV, BS = 2, 4, 96, 48, 8


def _batches(t, n_tiles, tile_bs):
    return [t[i * N:min(i + tile_bs, n_tiles) * N].clone() for i in range(0, n_tiles, tile_bs)]


def blends(L, frac, iters):
    g = engine.make_grid(L, L, TILE, TILE, OV, BS)
    x = torch.randn((N, C, L, L), device="cuda").half()
    tiles = engine.scatter_tiles(g, x)
    active = np.zeros(g.num_tiles, bool)
    active[np.random.default_rng(0).permutation(g.num_tiles)[:max(1, round(frac * g.num_tiles))]] = True
    idx = torch.tensor(np.flatnonzero(active), device="cuda")
    compact = tiles.view(g.num_tiles, N, C, TILE, TILE)[idx].reshape(-1, C, TILE, TILE)
    dense_outs, sparse_outs = _batches(tiles, g.num_tiles, g.tile_bs), _batches(compact, len(idx), g.tile_bs)
    slot = engine.slot_table(active)
    slot_dev = torch.from_numpy(slot).cuda()
    w_host = engine.grid_weights(g)
    w, rcp = torch.from_numpy(w_host).cuda(), torch.from_numpy(engine.exact_reciprocals(w_host)).cuda()
    gw = gaussian_weights(TILE, TILE).cuda()
    rf = torch.from_numpy(engine.rescale_factor(engine.grid_weights(g, gw.cpu().numpy()))).cuda()
    xo = torch.empty((N, C, L, L), dtype=torch.float32, device="cuda")
    xb = torch.empty((N, C, L, L), dtype=torch.float16, device="cuda")
    row = dict(latent=L, tiles=g.num_tiles, active=int(active.sum()))
    row["md_dense_us"] = round(time_us(lambda: engine.blend_multidiffusion(g, dense_outs, N, C, g.tile_bs, w, x.dtype, out=xo, rcp_weights=rcp),
                                       iters), 2)
    row["md_sparse_us"] = round(time_us(lambda: engine.blend_multidiffusion_sparse(g, sparse_outs, N, C, g.tile_bs, w, x.dtype, slot_dev, slot,
                                                                                   rcp_weights=rcp), iters), 2)
    row["mod_dense_us"] = round(time_us(lambda: engine.blend_mixture(g, dense_outs, N, C, g.tile_bs, gw, rf, xb), iters), 2)
    row["mod_sparse_us"] = round(time_us(lambda: engine.blend_mixture_sparse(g, sparse_outs, N, C, g.tile_bs, gw, rf, xb, slot_dev, slot),
                                         iters), 2)
    return row


def unet_calls(L):
    g = engine.make_grid(L, L, TILE, TILE, OV, BS)
    mask = torch.ones((L, L), device="cuda")
    c = L // 2
    mask[c - 64:c + 64, c - 64:c + 64] = 0
    n = int(engine.active_tiles(g, mask).sum())
    return dict(latent=L, tiles=g.num_tiles, active_tiles=n, unet_calls_full=int(g.num_batches), unet_calls_masked=-(-n // g.tile_bs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_inpaint_mask measures on the GPU"
    print(json.dumps({"card": card()}))
    for L in (512, 1024):
        print(json.dumps(unet_calls(L)))
        for frac in (0.1, 0.5, 1.0):
            print(json.dumps(dict(blends(L, frac, args.iters), fraction=frac)))


if __name__ == "__main__":
    main()
