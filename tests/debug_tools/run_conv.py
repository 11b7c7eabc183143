"""Hand-run launcher for ncu captures of the wgmma convolution (GPU box).
Usage: python tests/debug_tools/run_conv.py H W Cin Cout k [reps] [mode]
mode: plain (bias only) | gn (frozen GroupNorm + SiLU epilogue) | res (residual) | gnres | dual (residual, two outputs) | up (folded upsample)"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops as ops  # noqa: E402

H, W, Cin, Cout, k = (int(v) for v in sys.argv[1:6])
reps = int(sys.argv[6]) if len(sys.argv) > 6 else 3
mode = sys.argv[7] if len(sys.argv) > 7 else "plain"
x = (torch.randn((1, H, W, Cin), device="cuda") * 0.5).half()
b = torch.zeros(Cout, device="cuda")
post = (torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda"), True) if mode in ("gn", "gnres", "dual", "up") else None
if mode == "up":
    w = (torch.randn((16, Cout, Cin), device="cuda") * 0.02).half()
    for _ in range(reps):
        ops.upconv2x_nhwc(x, w, b, post=post)
else:
    w = (torch.randn((k * k, Cout, Cin), device="cuda") * 0.02).half()
    res = (torch.randn((1, H, W, Cout), device="cuda") * 0.5).half() if mode in ("res", "gnres", "dual") else None
    y = torch.empty((1, H, W, Cout), device="cuda", dtype=torch.float16)
    for _ in range(reps):
        ops.conv2d_nhwc(x, w, b, ksize=k, pad=(k // 2, k // 2), out=y, residual=res, post=post, dual=(mode == "dual"))
torch.cuda.synchronize()
print("ok")
