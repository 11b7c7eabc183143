"""Hand-run timing of the tiled VAE's mid-block attention (GPU box): the four-GEMM path against the fused kernel
(vae_ops.attention) per token count, then whole VAEHook calls of the full-width SD network (fp16, fast mode) at the
reference's tile sizes.  Prints the card and its power limit first; one JSON line per measurement.

    python tests/debug_tools/bench_attention.py [--iters 20] [--skip-hook]

Attention: TFLOP/s from 4 T^2 C (Q K^T and P V); peak = the rise of torch.cuda.max_memory_allocated() over the call,
q / k / v (and for the four-GEMM path V^T) allocated before.  The four-GEMM path is timed up to 45 796 tokens, the fused
kernel at every size."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from multidiffusion_upscaler_for_automatic1111_b200 import tilevae, vae_ops as ops  # noqa: E402
from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve  # noqa: E402

C = 512
BOTH = [13924, 32400, 45796]
FUSED_ONLY = [77284, 121104, 285156]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def four_gemm(q, k, vt, alpha, T):
    Tp = vt.shape[1]
    s = torch.empty((T, Tp), dtype=q.dtype, device=q.device)
    ops.gemm_nt(q, k, alpha=alpha, out=s[:, :T])
    ops.softmax_rows(s, T, out=s)
    return ops.gemm_nt(s, vt)


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, torch.cuda.max_memory_allocated() - base


def bench_attention(iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    alpha = C ** -0.5
    for T in BOTH + FUSED_ONLY:
        q = (torch.randn((T, C), generator=g, device="cuda") * 1.7).half()
        k = (torch.randn((T, C), generator=g, device="cuda") * 1.7).half()
        v = torch.randn((T, C), generator=g, device="cuda").half()
        flop = 4.0 * T * T * C
        n = max(3, iters * 13924 ** 2 // T ** 2)
        paths = [("fused", lambda: ops.attention(q, k, v, alpha))]
        if T in BOTH:
            Tp = ops.round_up(T, 8)
            vt = torch.zeros((C, Tp), dtype=torch.float16, device="cuda")
            vt[:, :T] = v.T
            paths.insert(0, ("four_gemm", lambda: four_gemm(q, k, vt, alpha, T)))
        for name, fn in paths:
            ms, peak = timed(fn, n)
            print(json.dumps({"what": "attention", "path": name, "tokens": T, "C": C, "iters": n, "ms": round(ms, 3),
                              "tflops": round(flop / ms / 1e9, 1), "peak_alloc_gib": round(peak / 2 ** 30, 3)}), flush=True)
        del q, k, v
        torch.cuda.empty_cache()


def bench_hook():
    from oracle import ldm_vae, synth
    runs = [(True, (1, 4, 1024, 1024), t) for t in (96, 256, 512)] + [(False, (1, 3, 8192, 8192), t) for t in (1536, 3072, 4096)]
    nets = {}
    for is_dec, shape, tile in runs:
        if is_dec not in nets:
            nets.clear()
            torch.cuda.empty_cache()
            net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), 3 if is_dec else 4).eval()
            net.original_forward = net.forward
            nets[is_dec] = net.cuda().half()
        x = synth.latent(5, shape, torch.float16).cuda()
        hook = tilevae.VAEHook(nets[is_dec], tile, is_dec, True, True, False)
        calls = []
        real = ve.ops.attention

        def spy(q, *a, **kw):
            calls.append(q.shape[0])
            return real(q, *a, **kw)
        ve.ops.attention = spy
        try:
            with torch.no_grad():
                hook(x)                                  # warm-up: weights packed, kernels loaded
                torch.cuda.synchronize()
                calls.clear()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                t0 = time.perf_counter()
                out = hook(x)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
        finally:
            ve.ops.attention = real
        print(json.dumps({"what": "vaehook", "decoder": is_dec, "input": list(shape), "tile": tile, "backend": hook.backend_name,
                          "fused_attention_calls": len(calls), "max_fused_tokens": max(calls) if calls else 0,
                          "wall_s": round(wall, 3), "peak_alloc_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2),
                          "finite": bool(torch.isfinite(out).all())}), flush=True)
        del out, x
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--skip-hook", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps({"card": card()}), flush=True)
    bench_attention(args.iters)
    if not args.skip_hook:
        bench_hook()


if __name__ == "__main__":
    main()
