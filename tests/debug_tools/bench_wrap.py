"""Seamless tiling: time the wrap scatter and blends (csrc/td_wrap.cu) against the bounded defaults on the same shapes.

    python tests/debug_tools/bench_wrap.py [--iters 2000]

Shapes: cfg2 ([2,4,512,512] fp16, tile 96, overlap 48: wrap xy is 11 x 11 = 121 tiles) and a panorama latent
[2,4,512,2048] wrapped in x; and a cfg4-size tiled VAE decode (z [1,4,1024,1024] -> 8192 x 8192, fp16, SD-width
decoder with seeded weights, tile 96, fast mode as bench.py's cfg4) with and without wrap in x and y.  Times are CUDA events around replays of a CUDA graph holding 20 calls (after a warm-up); algorithmic bytes
are computed from the shapes (tiles read or written once, canvas fp32 output, weights / rescale once) and set against
3.35 TB/s (H100 SXM data sheet).  Prints the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from multidiffusion_upscaler_for_automatic1111_b200 import engine  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:    # noqa: BLE001 - the name alone still identifies the card
        return torch.cuda.get_device_name()


def time_us(fn, iters, per_graph=20):
    """Kernel time per call: `per_graph` calls captured in one CUDA graph, replayed, timed with events.  Timing the Python
    calls directly would measure the host's launch rate (a ctypes call costs more than these kernels)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            fn()
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


def run_shape(name, N, C, H, W, tile, overlap, bs, wrap, iters):
    dt = torch.float16
    x = torch.randn((N, C, H, W), device="cuda").to(dt)
    res = []
    for label, wr in (("bounded", 0), ("wrap", wrap)):
        g = engine.make_grid(W, H, tile, tile, overlap, bs, wrap=wr)
        T = g.num_tiles
        tiles = engine.scatter_tiles(g, x)
        outs = [tiles[b * g.tile_bs * N:min((b + 1) * g.tile_bs, T) * N].clone() for b in range(g.num_batches)]
        w_host = engine.grid_weights(g)
        wts = torch.from_numpy(w_host).cuda()
        rcp = engine.exact_reciprocals(w_host)
        rcp = torch.from_numpy(rcp).cuda() if rcp is not None else None
        from oracle import tiling
        tw_host = tiling.gaussian_weights(g.tile_w, g.tile_h)
        gw = engine.grid_weights(g, tw_host)
        rescale = torch.from_numpy(engine.rescale_factor(gw)).cuda()
        tw_dev = torch.from_numpy(tw_host).cuda()
        xbuf = torch.empty_like(x)
        out = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")
        tile_bytes = T * N * C * g.tile_h * g.tile_w * 2
        canvas16, canvas32, plane32 = N * C * H * W * 2, N * C * H * W * 4, H * W * 4
        cases = {
            "scatter": (lambda: engine.scatter_tiles(g, x, out=tiles), tile_bytes + canvas16),
            "md_blend": (lambda: engine.blend_multidiffusion(g, outs, N, C, g.tile_bs, wts, dt, out=out, rcp_weights=rcp),
                         tile_bytes + canvas32 + plane32),
            "mod_blend": (lambda: engine.blend_mixture(g, outs, N, C, g.tile_bs, tw_dev, rescale, xbuf), tile_bytes + canvas16 + plane32),
        }
        for op, (fn, nbytes) in cases.items():
            us = time_us(fn, iters)
            bound = nbytes / PEAK_BPS * 1e6
            res.append(dict(shape=name, form=label, op=op, tiles=T, us=round(us, 2), mbytes=round(nbytes / 1e6, 2),
                            bound_us=round(bound, 2), share_of_hbm_bound=round(bound / us, 3)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--no-vae", action="store_true", help="skip the cfg4-size VAE decode")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wrap measures on the GPU"
    print(json.dumps({"card": card()}))
    rows = run_shape("cfg2 [2,4,512,512]", 2, 4, 512, 512, 96, 48, 4, engine.WRAP_X | engine.WRAP_Y, args.iters)
    rows += run_shape("panorama [2,4,512,2048]", 2, 4, 512, 2048, 96, 48, 4, engine.WRAP_X, args.iters)
    for r in rows:
        print(json.dumps(r))
    if not args.no_vae:
        print(json.dumps(vae_decode()))


def vae_decode():
    """cfg4-size decode, bounded vs wrapped (one warm-up call each, then one timed call each, alternated)."""
    import time

    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from oracle import ldm_vae, synth
    net = ldm_vae.seeded_init(ldm_vae.Decoder(), 3).eval().half().cuda()
    net.original_forward = net.forward
    z = synth.latent(5, (1, 4, 1024, 1024), torch.float16).cuda()
    hook = tilevae.VAEHook(net, 96, True, fast_decoder=True, fast_encoder=True, color_fix=False)   # bench.py's cfg4 default
    times = {"bounded": [], "wrap_xy": []}
    with torch.no_grad():
        for rep in range(2):
            for label, w in (("bounded", False), ("wrap_xy", True)):
                hook.wrap_x = hook.wrap_y = w
                torch.cuda.empty_cache()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                hook(z)
                torch.cuda.synchronize()
                if rep:
                    times[label].append(time.perf_counter() - t0)
    tiles = {}
    hook.wrap_x = hook.wrap_y = True
    tiles["wrap_xy"] = len(hook.split_tiles(1024, 1024)[0])
    hook.wrap_x = hook.wrap_y = False
    tiles["bounded"] = len(hook.split_tiles(1024, 1024)[0])
    return {"vae_decode_8192": {k: round(v[0], 3) for k, v in times.items()}, "tiles": tiles, "backend": hook.backend_name}


if __name__ == "__main__":
    main()
