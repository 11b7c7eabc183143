"""The strip form of the MultiDiffusion blend (csrc/td_strip.cu, TD_FLAG_STRIP) executed on the HOST: the kernel's three
phases are __host__ __device__ functions, a test-only harness runs every CTA thread by thread over an emulated shared
memory, and the result must be bit-identical to the fixtures generated from the unmodified reference.  This pins the
staging layout, the index arithmetic and the rounding sequence of a kernel that has not run on hardware yet."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from helpers import load_golden, DTYPES, assert_bit_equal, sha
from oracle import blend, synth, tiling
from oracle.make_golden import BLEND_CASES, HASH_CASES

PKG = os.path.join(ROOT, "multidiffusion_upscaler_for_automatic1111_b200")
ROWS = int(os.environ.get("TD_STRIP_ROWS", "8"))      # the kernel's tuning knob; run the file with another value to check a variant
CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out_dir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"libtd_strip_emul_r{ROWS}.so")
    srcs = [os.path.join(ROOT, "tests", "emul", "strip_host_emul.cu"), os.path.join(PKG, "csrc", "td_host.cpp")]
    deps = srcs + [os.path.join(PKG, "csrc", "td_strip.cu"), os.path.join(PKG, "csrc", "td_device.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
               "--expt-relaxed-constexpr", f"-DTD_STRIP_ROWS={ROWS}", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(PKG, "csrc"),
               "-o", so, *srcs]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-3000:]
    return ctypes.CDLL(so)


def _strip_step(emul, x, W, H, tw, th, ov, bs, use_rcp=False, want_buffer=True, max_ppc=2):
    """scatter (oracle) -> fake UNet per batch -> emulated strip blend.  Returns (x_out fp32, x_buffer, launch info)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N, C = x.shape[:2]
    g = engine.make_grid(W, H, tw, th, ov, bs)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, False)
    outs = [synth.fake_denoise(blend.scatter_tiles(x, bbs), bbs, N).contiguous() for bbs in plan.batched_bboxes]
    ptrs = (ctypes.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    weights = np.ascontiguousarray(plan.weights, dtype=np.float32)
    rcp = engine.exact_reciprocals(weights) if use_rcp else None
    x_out = torch.empty((N, C, H, W), dtype=torch.float32)
    xb = torch.empty_like(x) if want_buffer else None
    info = (ctypes.c_int * 4)()
    rc = emul.td_emul_strip_blend(ctypes.byref(g), ptrs, len(outs), int(g.tile_bs), N, C, CODE[x.dtype],
                                  weights.ctypes.data_as(ctypes.c_void_p), rcp.ctypes.data_as(ctypes.c_void_p) if rcp is not None else None,
                                  ctypes.c_void_p(x_out.data_ptr()), ctypes.c_void_p(xb.data_ptr()) if xb is not None else None, max_ppc, info)
    return rc, x_out, xb, tuple(info), plan


@pytest.mark.parametrize("case", BLEND_CASES, ids=[c[0] for c in BLEND_CASES])
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("max_ppc", [1, 2], ids=["one_plane", "two_planes"])
def test_emulated_strip_blend_matches_reference_fixture(emul, golden_dir, case, dn, max_ppc):
    name, N, C, W, H, tw, th, ov, bs = case
    dt = DTYPES[dn]
    x = synth.latent(synth.case_seed(name, dn), (N, C, H, W), dt)
    vec = 16 // x.element_size()
    rc, x_out, xb, info, plan = _strip_step(emul, x, W, H, tw, th, ov, bs, max_ppc=max_ppc)
    if W % vec or min(tw, W) % vec:
        assert rc == 1                                   # not applicable: the entry point falls back to the default kernels
        return
    assert rc == 0 and info[3] == (max_ppc if (N * C) % 2 == 0 else 1)
    g = load_golden(golden_dir, "blend_small")
    want = torch.from_numpy(g[f"{name}_{dn}_md"].view(np.int32).copy()).view(torch.float32)
    assert_bit_equal(x_out, want, "strip blend vs reference")
    # x_buffer is the un-normalised accumulator of the reference (multidiffusion.py:166-167)
    acc = torch.zeros_like(x)
    for bbs in plan.batched_bboxes:
        blend.accumulate_md(acc, synth.fake_denoise(blend.scatter_tiles(x, bbs), bbs, N), bbs, N)
    assert_bit_equal(xb, acc, "strip x_buffer")


@pytest.mark.parametrize("dn", ["f16", "bf16"])
def test_emulated_strip_blend_with_exact_reciprocals(emul, golden_dir, dn):
    name, N, C, W, H, tw, th, ov, bs = BLEND_CASES[4]      # the UI default tile on a small canvas
    x = synth.latent(synth.case_seed(name, dn), (N, C, H, W), DTYPES[dn])
    rc, x_out, _, info, _ = _strip_step(emul, x, W, H, tw, th, ov, bs, use_rcp=True, want_buffer=False)
    assert rc == 0
    g = load_golden(golden_dir, "blend_small")
    want = torch.from_numpy(g[f"{name}_{dn}_md"].view(np.int32).copy()).view(torch.float32)
    assert_bit_equal(x_out, want, "strip blend, fast exact divide")


def test_emulated_strip_blend_full_size_cfg2(emul, golden_dir):
    """BASELINE cfg2 (512 x 512 latent, 100 tiles): sha256 of the reference's output, and the launch shape the design
    argues with -- 64 strips x 8 planes = 512 CTAs of 512 threads, ~54 KB of shared memory each (one wave on 132 SMs)."""
    name, N, C, W, H, tw, th, ov, bs = HASH_CASES[0]
    x = synth.latent(synth.case_seed(name, "f16"), (N, C, H, W), torch.float16)
    rc, x_out, _, info, _ = _strip_step(emul, x, W, H, tw, th, ov, bs, use_rcp=True, want_buffer=False)
    assert rc == 0
    strips, nthreads, smem, ppc = info
    assert (strips, nthreads, ppc) == (-(-512 // ROWS), ROWS * 64, 2)
    if ROWS == 8:
        assert 100_000 < smem < 112_000      # two planes per CTA: 2 CTAs / SM, 256 CTAs -> still one wave on 132 SMs
    g = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
    assert sha(x_out) == str(g[f"{name}_f16_md"])


@pytest.mark.parametrize("geom", [(2, 4, 160, 64, 96, 96, 48, 2), (1, 4, 64, 160, 200, 48, 16, 1), (2, 4, 72, 72, 24, 16, 6, 3),
                                  (1, 2, 1024, 40, 96, 32, 4, 8)])
def test_emulated_strip_blend_edge_geometries(emul, geom):
    N, C, W, H, tw, th, ov, bs = geom
    x = synth.latent(5, (N, C, H, W), torch.float16)
    rc, x_out, xb, info, plan = _strip_step(emul, x, W, H, tw, th, ov, bs)
    if ROWS * (W // 8) > 1024:
        assert rc == 1                                   # more than 1024 threads per strip: not applicable, default kernels run
        return
    assert rc == 0
    want = blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, lambda t, bb: synth.fake_denoise(t, bb, N))
    assert_bit_equal(x_out, want, f"strip blend {geom}")


# ------------------------------------------------------------------------------------------ Mixture of Diffusers on strips
def _strip_step_mod(emul, x, W, H, tw, th, ov, bs):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N, C = x.shape[:2]
    g = engine.make_grid(W, H, tw, th, ov, bs)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, True)
    outs = [synth.fake_denoise(blend.scatter_tiles(x, bbs), bbs, N).contiguous() for bbs in plan.batched_bboxes]
    ptrs = (ctypes.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    twt = np.ascontiguousarray(plan.tile_weights, dtype=np.float32)
    rf = np.ascontiguousarray(plan.rescale_factor, dtype=np.float32)
    xb = torch.empty_like(x)
    rc = emul.td_emul_strip_blend_mod(ctypes.byref(g), ptrs, len(outs), int(g.tile_bs), N, C, CODE[x.dtype],
                                      twt.ctypes.data_as(ctypes.c_void_p), rf.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(xb.data_ptr()))
    return rc, xb


@pytest.mark.parametrize("case", BLEND_CASES, ids=[c[0] for c in BLEND_CASES])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_emulated_strip_mixture_matches_reference_fixture(emul, golden_dir, case, dn):
    name, N, C, W, H, tw, th, ov, bs = case
    x = synth.latent(synth.case_seed(name, dn), (N, C, H, W), DTYPES[dn])
    vec = 16 // x.element_size()
    rc, xb = _strip_step_mod(emul, x, W, H, tw, th, ov, bs)
    if W % vec or min(tw, W) % vec:
        assert rc == 1
        return
    assert rc == 0
    g = load_golden(golden_dir, "blend_small")
    raw = g[f"{name}_{dn}_mod"]
    want = torch.from_numpy(raw.view(np.int16 if raw.dtype == np.uint16 else np.int32).copy()).view(DTYPES[dn])
    from helpers import bits
    assert np.array_equal(bits(xb), raw), f"{name} {dn}: strip Mixture of Diffusers differs from the reference's (sign of zero included)"
    assert_bit_equal(xb, want, "strip mixture vs reference")


def test_emulated_strip_mixture_full_size_cfg2(emul, golden_dir):
    name, N, C, W, H, tw, th, ov, bs = HASH_CASES[0]
    x = synth.latent(synth.case_seed(name, "f16"), (N, C, H, W), torch.float16)
    rc, xb = _strip_step_mod(emul, x, W, H, tw, th, ov, bs)
    assert rc == 0
    g = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
    assert sha(xb) == str(g[f"{name}_f16_mod"])
