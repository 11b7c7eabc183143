"""Masked against unmasked cfg4 decode, and the td_vae_active_tiles pass against the HBM bound.

    python tests/debug_tools/bench_vae_inpaint.py [--reps 3]

Workload: the SD-width decoder (seeded), z [1, 4, 1024, 1024] fp16, tile 96 (121 tiles of an 8192 x 8192 image), fast mode,
with a 1024 x 1024 image-space square in the middle to inpaint (mask 0 inside, 1 outside, fill = a constant image).  The
fast-mode estimate runs in both calls, so the masked call saves less than the tile ratio.  Prints one JSON line: the GPU and
its power limit, the tiles the mask reaches (counted from the split on the host), the wall time of each call (median of
--reps, masked and unmasked alternating), whether the active rectangles are bit-identical, and the active-tiles kernel time
(CUDA events over 50 launches) against 134 MB at 3.35 TB/s.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from multidiffusion_upscaler_for_automatic1111_b200 import engine, tilevae  # noqa: E402
from oracle import ldm_vae, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:     # noqa: BLE001
        q = f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"
    return q


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    torch.cuda.set_device(0)
    net = ldm_vae.seeded_init(ldm_vae.Decoder(), 3).eval()
    net.original_forward = net.forward
    net = net.cuda().half()
    hook = tilevae.VAEHook(net, 96, True, fast_decoder=True, fast_encoder=True, color_fix=False)
    z = synth.latent(1, (1, 4, 1024, 1024), torch.float32).cuda().half()
    oh = ow = 8192
    mask = torch.ones(oh, ow, dtype=torch.float16, device="cuda")
    mask[oh // 2 - 512:oh // 2 + 512, ow // 2 - 512:ow // 2 + 512] = 0.0
    fill = torch.full((1, 3, oh, ow), -0.5, dtype=torch.float16, device="cuda")
    rects = hook.split_tiles(1024, 1024)[1]
    active_host = np.array([(mask[b[2]:b[3], b[0]:b[1]] != 1).any().item() for b in rects])

    def plain():
        hook.set_inpaint_mask(None)
        with torch.no_grad():
            return hook(z)

    def masked():
        hook.set_inpaint_mask(mask, fill)
        try:
            with torch.no_grad():
                return hook(z)
        finally:
            hook.set_inpaint_mask(None)

    want, _ = timed(plain)          # warm-up of every shape both calls use
    got, _ = timed(masked)
    stats = dict(hook.last_park_stats)
    same = all(torch.equal(got[:, :, b[2]:b[3], b[0]:b[1]], want[:, :, b[2]:b[3], b[0]:b[1]]) for b, a in zip(rects, active_host) if a)
    kept = all(torch.equal(got[:, :, b[2]:b[3], b[0]:b[1]], fill[:, :, b[2]:b[3], b[0]:b[1]]) for b, a in zip(rects, active_host) if not a)
    del got, want
    t_plain, t_masked = [], []
    for _ in range(args.reps):
        t_plain.append(timed(plain)[1])
        t_masked.append(timed(masked)[1])

    engine.vae_active_tiles(mask, rects)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    launches = 50
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import check, current_stream_ptr, dtype_code, lib
    import ctypes
    r = np.ascontiguousarray(np.asarray(rects, dtype=np.int32))
    out = torch.empty(len(rects), dtype=torch.uint8, device="cuda")
    m1 = torch.ones_like(mask)      # all keep: every CTA reads its rows (no early exit)
    call = lambda mk: check(lib.td_vae_active_tiles(mk.data_ptr(), 1, oh, ow, dtype_code(mk.dtype), r.ctypes.data_as(
        ctypes.POINTER(ctypes.c_int32)), len(rects), out.data_ptr(), current_stream_ptr()))
    call(m1)
    ev[0].record()
    for _ in range(launches):
        call(m1)
    ev[1].record()
    torch.cuda.synchronize()
    kernel_s = ev[0].elapsed_time(ev[1]) / 1e3 / launches
    nbytes = sum((b[1] - b[0]) * (b[3] - b[2]) for b in rects) * 2
    print(json.dumps({
        "gpu": gpu_info(), "tiles": len(rects), "tiles_reached": int(active_host.sum()), "tiles_run": stats["tiles_run"],
        "tiles_skipped": stats["tiles_skipped"], "unmasked_s": float(np.median(t_plain)), "masked_s": float(np.median(t_masked)),
        "unmasked_all_s": t_plain, "masked_all_s": t_masked, "speedup": float(np.median(t_plain) / np.median(t_masked)),
        "active_bit_identical": bool(same), "skipped_equal_fill": bool(kept),
        "active_tiles_kernel_us": kernel_s * 1e6, "active_tiles_bytes": nbytes,
        "active_tiles_share_of_hbm_bound": nbytes / HBM_BYTES_PER_S / kernel_s,
    }))


if __name__ == "__main__":
    main()
