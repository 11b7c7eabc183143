"""Hand-run measurement of slow-mode tile parking (GPU box): tiled decodes whose GroupNorm barriers hold more than the
GPU's memory, and cfg4's decode with budgets that force parking.  Prints the card and its power limit first, then one
JSON line per run: wall time, peak allocated HBM, pinned host bytes, bytes copied each way and the achieved GB/s per
direction (bytes / wall time: a lower bound on the copy engines' rate, since copies overlap with compute).

    python tests/debug_tools/bench_vae_park.py [--skip-large] [--skip-cfg4]

Runs (full-width SD decoder, synthetic weights, tile 96, slow mode):
  * fp16 z [1, 4, 1536, 1536] -> 12288^2 (256 tiles; 171 GB at the widest barrier);
  * fp32 z [1, 4, 1024, 1024] -> 8192^2 on the module backend (121 tiles; 152 GB);
  * cfg4 fp16 z [1, 4, 1024, 1024]: unbounded, then budgets that park about half and all of the tiles; the three
    outputs are compared byte for byte.  cfg4's fast and slow decodes at the default budget must park nothing."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from multidiffusion_upscaler_for_automatic1111_b200 import tilevae, vae_engine as ve  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def decoder(dtype):
    from oracle import ldm_vae
    net = ldm_vae.seeded_init(ldm_vae.Decoder(), 1).eval()
    net.original_forward = net.forward
    return net.cuda().to(dtype)


def barrier_peak(hook, lat, dtype):
    prog = ve.compile_program(hook.net, True)
    name = ve.pick_backend(prog, torch.device("cuda"), dtype).name
    ib, _ = hook.split_tiles(lat, lat)
    fps = [ve.tile_footprint(prog, name, dtype, b[3] - b[2], b[1] - b[0]) for b in ib]
    return max(sum(f.held(s) for f in fps) for s in range(prog.num_sites))


def run(label, hook, z, budget=None):
    hook.max_resident_bytes = budget
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    line = {"run": label, "input": list(z.shape), "dtype": str(z.dtype).replace("torch.", ""), "slow": not hook.fast_mode,
            "max_resident_bytes": budget, "host_mem_available_gb": round((ve.host_available_bytes() or 0) / 1e9, 1)}
    out = None
    t0 = time.perf_counter()
    try:
        with torch.no_grad():
            out = hook(z)
        torch.cuda.synchronize()
    except (RuntimeError, torch.OutOfMemoryError) as e:
        line.update(ok=False, error=str(e)[:300])
    wall = time.perf_counter() - t0
    st = hook.last_park_stats or {}
    line.update(wall_s=round(wall, 2), peak_hbm_gb=round((torch.cuda.max_memory_allocated() - base) / 1e9, 2),
                backend=hook.backend_name, budget_gb=None if st.get("budget") is None else round(st["budget"] / 1e9, 2),
                pinned_host_gb=round(st.get("host_bytes", 0) / 1e9, 2), pin_s=round(st.get("pin_s", 0.0), 2), d2h_gb=round(st.get("d2h_bytes", 0) / 1e9, 2),
                h2d_gb=round(st.get("h2d_bytes", 0) / 1e9, 2), tiles_parked=sum(st.get("tiles_parked", {}).values()),
                d2h_gbps=round(st.get("d2h_bytes", 0) / 1e9 / wall, 1), h2d_gbps=round(st.get("h2d_bytes", 0) / 1e9 / wall, 1))
    digest = None
    if out is not None:
        line.update(ok=True, finite=bool(torch.isfinite(out).all()))
        digest = hashlib.sha256(out.cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()
        line["sha256"] = digest[:16]
    print(json.dumps(line), flush=True)
    del out
    torch.cuda.empty_cache()
    return line, digest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-large", action="store_true")
    ap.add_argument("--skip-cfg4", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vae_park.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    print(json.dumps({"card": card(), "host_mem_available_gb": round((ve.host_available_bytes() or 0) / 1e9, 1)}), flush=True)
    g = torch.Generator().manual_seed(7)
    if not args.skip_large:
        net = decoder(torch.float16)
        z = torch.randn((1, 4, 1536, 1536), generator=g).half().cuda()
        run("fp16 slow decode 12288^2", tilevae.VAEHook(net, 96, True, False, False, False), z)
        del net, z
        net = decoder(torch.float32)
        z = torch.randn((1, 4, 1024, 1024), generator=torch.Generator().manual_seed(7)).cuda()
        run("fp32 slow decode 8192^2 (modules)", tilevae.VAEHook(net, 96, True, False, False, False), z)
        del net, z
        torch.cuda.empty_cache()
    if not args.skip_cfg4:
        net = decoder(torch.float16)
        z = torch.randn((1, 4, 1024, 1024), generator=torch.Generator().manual_seed(7)).half().cuda()
        fast = tilevae.VAEHook(net, 96, True, True, True, False)
        line, _ = run("cfg4 fast decode, default budget", fast, z)
        assert line.get("ok") and line["tiles_parked"] == 0, "cfg4 fast mode parked tiles"
        hook = tilevae.VAEHook(net, 96, True, False, False, False)
        peak = barrier_peak(hook, 1024, torch.float16)
        digests = []
        for label, budget in (("unbounded", None), ("~50% parked", peak // 2), ("100% parked", 0)):
            line, d = run(f"cfg4 slow decode, {label}", hook, z, budget)
            if budget is None:
                assert line.get("ok") and line["tiles_parked"] == 0, "cfg4 slow mode parked tiles at the default budget"
            digests.append(d)
        print(json.dumps({"cfg4_slow_outputs_identical": len(set(digests)) == 1 and digests[0] is not None}), flush=True)


if __name__ == "__main__":
    main()
