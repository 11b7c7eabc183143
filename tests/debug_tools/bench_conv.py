"""Hand-run timing of the wgmma convolution at BASELINE cfg4's decoder shapes (GPU box): TFLOP/s of td_conv2d_nhwc
next to cuDNN (F.conv2d, channels_last fp16) on the same tensors.  Usage: python tests/debug_tools/bench_conv.py"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops as ops  # noqa: E402


def timeit(fn, reps):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def main():
    out = {}
    shapes = [(944, 944, 128, 128, 3), (944, 944, 256, 128, 3), (472, 472, 256, 256, 3), (472, 472, 512, 256, 3),
              (236, 236, 512, 512, 3), (118, 118, 512, 512, 3), (944, 944, 128, 16, 3), (472, 472, 512, 256, 1)]
    if len(sys.argv) > 1 and sys.argv[1] == "--quick":
        shapes = [shapes[0]] + shapes[2:6]
    for (H, W, Cin, Cout, k) in shapes:
        x = (torch.randn((1, H, W, Cin), device="cuda") * 0.5).half()
        w = (torch.randn((k * k, Cout, Cin), device="cuda") * 0.02).half()
        b = torch.zeros(Cout, device="cuda")
        y = torch.empty((1, H, W, Cout), device="cuda", dtype=torch.float16)
        flops = 2.0 * H * W * Cin * Cout * k * k
        t = timeit(lambda: ops.conv2d_nhwc(x, w, b, ksize=k, pad=(k // 2, k // 2), out=y), 5)
        xc = x.permute(0, 3, 1, 2)   # channels_last view
        wc = w.view(k, k, Cout, Cin).permute(2, 3, 0, 1).contiguous(memory_format=torch.channels_last)
        tc = timeit(lambda: F.conv2d(xc, wc, None, padding=k // 2), 5)
        ref = F.conv2d(xc, wc, None, padding=k // 2)
        err = (y.permute(0, 3, 1, 2).float() - ref.float()).abs().max().item() / (ref.float().abs().max().item() + 1e-9)
        out[f"{H}x{W} {Cin}->{Cout} k{k}"] = {"ours_ms": round(t * 1e3, 4), "ours_tflops": round(flops / t / 1e12, 1),
                                             "cudnn_ms": round(tc * 1e3, 4), "cudnn_tflops": round(flops / tc / 1e12, 1), "rel_err_vs_cudnn": err}
        print(json.dumps({f"{H}x{W} {Cin}->{Cout} k{k}": out[f"{H}x{W} {Cin}->{Cout} k{k}"]}), flush=True)
    # attention GEMMs of one decoder tile: 13924 tokens, C = 512
    T, C = 13924, 512
    q = (torch.randn((T, C), device="cuda") * 0.3).half()
    kk = (torch.randn((T, C), device="cuda") * 0.3).half()
    pitch = ops.round_up(T, 8)
    s = torch.empty((T, pitch), device="cuda", dtype=torch.float16)
    t = timeit(lambda: ops.gemm_nt(q, kk, alpha=C ** -0.5, out=s[:, :T]), 3)
    print(json.dumps({"attn QK^T 13924x512x13924": {"ms": round(t * 1e3, 3), "tflops": round(2.0 * T * T * C / t / 1e12, 1)}}), flush=True)
    tm = timeit(lambda: torch.matmul(q, kk.t()), 3)
    print(json.dumps({"cublas QK^T": {"ms": round(tm * 1e3, 3), "tflops": round(2.0 * T * T * C / tm / 1e12, 1)}}), flush=True)


if __name__ == "__main__":
    main()
