"""Seamless DemoFusion: time one `sample_one_step` bounded vs wrapped in x vs wrapped in x and y, on the grid and with random
jitter, and the gaussian stencil td_depthwise_conv2d against td_depthwise_conv2d_wrap on the same tensor.

    python tests/debug_tools/bench_demofusion_wrap.py [--steps 20] [--rounds 5] [--out results/demofusion_wrap.json]

Geometry: BASELINE cfg5 (bench.py's DEMO: latent [2,4,768,768], window 128, stride 64, scale 4, mixture, identity UNet
stand-in), fp16 and bf16.  The bounded grid has 11 x 11 = 121 windows, the wrap-xy grid 12 x 12 = 144.  Bounded jitter
steps the latent padded by jitter_range (as forward_one_step hands it over); the wrapped ones step the latent itself.
The variants alternate within each round, after a warm-up of every one; a round times `steps` consecutive steps with
CUDA events.  Reported: the median over rounds of the per-step time, and the card name and power limit read in the run.
"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..")
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi  # noqa: E402
from oracle import demofusion as odf  # noqa: E402
from oracle import synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:    # noqa: BLE001 - the name alone still identifies the card
        return torch.cuda.get_device_name()


def step_fn(dt, jitter, wrap_x, wrap_y):
    c = bench.DEMO
    d, fwd, _ = bench._demo_job(torch.device("cuda"), dt, True, jitter)
    d.sampler_forward = fwd
    random.seed(1234)
    d.get_views(c["overlap"], c["tile_bs"], c["tile_bs_g"], wrap_x=wrap_x, wrap_y=wrap_y)
    d.cosine_factor = odf.cosine_factor(c["current_step"], c["t_enc"])
    pad = d.jitter_range if jitter and not (wrap_x or wrap_y) else 0
    L = c["lat"]
    x = synth.latent(5, (c["N"], c["C"], L, L), dt).cuda()
    x = torch.nn.functional.pad(x, (pad, pad, pad, pad)) if pad else x
    sigma = torch.ones(c["N"], device="cuda")
    cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8, device="cuda")], "c_concat": [torch.zeros(c["N"], 5, 1, 1, device="cuda")]}
    return (lambda: d.sample_one_step(x, sigma, cond)), d.num_tiles


def conv_fn(dt, wrap):
    c = bench.DEMO
    L, s = c["lat"], c["scale"]
    x = synth.latent(6, (c["N"], c["C"], L, L), dt).cuda()
    out = torch.empty_like(x)
    k = 2 * s - 1
    w = np.ascontiguousarray(odf.gaussian_kernel(k, 0.6, 1)[0, 0].to(dt).float().numpy())
    wp = w.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    planes, st = c["N"] * c["C"], _cabi.current_stream_ptr()
    if wrap is None:
        return lambda: _cabi.check(_cabi.lib.td_depthwise_conv2d(x.data_ptr(), out.data_ptr(), planes, L, L, wp, k, _cabi.dtype_code(dt), st))
    return lambda: _cabi.check(_cabi.lib.td_depthwise_conv2d_wrap(x.data_ptr(), out.data_ptr(), planes, L, L, wp, k, wrap,
                                                                  _cabi.dtype_code(dt), st))


def time_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--conv-iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {"card": card(), "steps": args.steps, "rounds": args.rounds, "step_ms": {}, "conv_us": {}, "windows": {}}
    for dt in (torch.float16, torch.bfloat16):
        dn = str(dt).split(".")[-1]
        variants = {}
        for jitter in (False, True):
            for name, wx, wy in (("bounded", False, False), ("wrap_x", True, False), ("wrap_xy", True, True)):
                key = f"{dn}/{'jitter' if jitter else 'grid'}/{name}"
                variants[key], result["windows"][key] = step_fn(dt, jitter, wx, wy)
        convs = {f"{dn}/td_depthwise_conv2d": conv_fn(dt, None), f"{dn}/td_depthwise_conv2d_wrap(xy)": conv_fn(dt, 3)}
        for fn in list(variants.values()) + list(convs.values()):   # warm-up: every shape, module load, allocator
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in list(variants) + list(convs)}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                times[k].append(time_ms(fn, args.steps))
            for k, fn in convs.items():
                times[k].append(time_ms(fn, args.conv_iters) * 1e3)
        for k in variants:
            result["step_ms"][k] = round(float(np.median(times[k])), 3)
        for k in convs:
            result["conv_us"][k] = round(float(np.median(times[k])), 2)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
