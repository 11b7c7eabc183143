"""Hand-run measurement of the batched tensor-core VAE pass (GPU box): fp16 full-width SD decoder and encoder (synthetic
weights) on batches of N = 1, 2, 4 images, one pass per image (images_per_pass = 1) against the count VAEHook picks.
Prints the card, its power limit and SM clock first, then one JSON line per run: milliseconds per call (CUDA events
around the call, median of the timed calls, after a warm-up call), the images per pass, kernels launched per call and
per pass (CUPTI trace through torch.profiler, in a separate untimed call), and whether the output is bit-identical to
the one-image schedule.

    python tests/debug_tools/bench_vae_batch.py [--reps 5] [--slow]

Runs: decode z [N, 4, 128, 128] -> 1024^2 at tile 64 (4 tiles); encode an [N, 3, 1024, 1024] image at tile 512
(4 tiles).  Fast mode by default (the WebUI default), --slow adds slow mode."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from multidiffusion_upscaler_for_automatic1111_b200 import tilevae  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def network(is_dec):
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), 1 if is_dec else 2).eval()
    net.original_forward = net.forward
    return net.cuda().half()


def call(hook, x, k):
    hook.images_per_pass = k
    with torch.no_grad():
        return hook(x)


def time_ms(hook, x, k, reps):
    call(hook, x, k)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        call(hook, x, k)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def kernels(hook, x, k):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(hook, x, k)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(names), sum("conv_gemm_kernel" in n for n in names)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--slow", action="store_true")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    for is_dec in (True, False):
        net = network(is_dec)
        for fast in ((True, False) if args.slow else (True,)):
            hook = tilevae.VAEHook(net, 64 if is_dec else 512, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
            for N in (1, 2, 4):
                g = torch.Generator().manual_seed(N)
                shape = (N, 4, 128, 128) if is_dec else (N, 3, 1024, 1024)
                x = torch.randn(shape, generator=g).cuda().half()
                ref = call(hook, x, 1)
                for k in ((1, None) if N > 1 else (1,)):
                    ms = time_ms(hook, x, k, args.reps)
                    out = call(hook, x, k)
                    chosen = hook.last_park_stats["images_per_pass"]
                    total, convs = kernels(hook, x, k)
                    passes = -(-N // chosen)
                    print(json.dumps({"run": "decode" if is_dec else "encode", "mode": "fast" if fast else "slow", "input": list(shape),
                                      "tiles": len(hook.split_tiles(shape[2], shape[3])[0]), "images_per_pass": chosen,
                                      "ms": round(ms, 2), "ms_per_image": round(ms / N, 2), "kernels": total,
                                      "kernels_per_pass": total // passes, "conv_launches_per_pass": convs // passes,
                                      "bit_identical_to_k1": bool(torch.equal(out.view(torch.int16), ref.view(torch.int16)))}),
                          flush=True)
                del x, ref, out
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
