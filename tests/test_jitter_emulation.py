"""The per-element bodies of csrc/td_jitter.cu (list-driven scatter / blend, offset combine) executed on the HOST by a
test-only harness (tests/emul/jitter_host_emul.cu, built here with nvcc) and compared bit for bit with torch: index
arithmetic and rounding sequence of kernels that have not run on hardware yet.  The product library has no host path."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from helpers import DTYPES
from oracle import synth

PKG = os.path.join(ROOT, "multidiffusion_upscaler_for_automatic1111_b200")
CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out_dir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libtd_jitter_emul.so")
    srcs = [os.path.join(ROOT, "tests", "emul", "jitter_host_emul.cu"), os.path.join(PKG, "csrc", "td_host.cpp")]
    deps = srcs + [os.path.join(PKG, "csrc", "td_jitter.cu")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
               "--expt-relaxed-constexpr", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(PKG, "csrc"), "-o", so, *srcs]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-3000:]
    return ctypes.CDLL(so)


def _origins(T, H, W, ws, seed):
    rng = np.random.default_rng(seed)
    org = [(int(rng.integers(0, W - ws + 1)), int(rng.integers(0, H - ws + 1))) for _ in range(T)]
    flat = np.array([v for o in org for v in o], dtype=np.int32)
    return org, flat


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("dn", list(DTYPES))
def test_emulated_scatter_and_blend_equal_eager(emul, dn):
    dt = DTYPES[dn]
    N, C, H, W, ws, tile_bs, T = 2, 3, 45, 70, 16, 4, 13
    org, flat = _origins(T, H, W, ws, 11)
    x = synth.latent(12, (N, C, H, W), dt).contiguous()
    tiles = torch.empty((T * N, C, ws, ws), dtype=dt)
    emul.td_emul_scatter_bboxes(_p(x), _p(tiles), flat.ctypes.data_as(ctypes.c_void_p), T, N, C, H, W, ws, ws, x.element_size())
    assert torch.equal(tiles, torch.cat([x[:, :, oy:oy + ws, ox:ox + ws] for ox, oy in org], dim=0))

    outs_src = synth.latent(13, (T * N, C, ws, ws), dt)
    nb = -(-T // tile_bs)
    outs = [outs_src[b * tile_bs * N:min((b + 1) * tile_bs, T) * N].contiguous() for b in range(nb)]
    ptrs = (ctypes.c_void_p * nb)(*[o.data_ptr() for o in outs])
    got = torch.empty((N, C, H, W), dtype=torch.float32)
    emul.td_emul_blend_bboxes(ptrs, nb, tile_bs, flat.ctypes.data_as(ctypes.c_void_p), T, N, C, H, W, ws, ws, CODE[dt], _p(got))
    buf, cnt = torch.zeros_like(x), torch.zeros_like(x)
    for t, (ox, oy) in enumerate(org):
        buf[:, :, oy:oy + ws, ox:ox + ws] += outs_src[t * N:(t + 1) * N]
        cnt[:, :, oy:oy + ws, ox:ox + ws] += 1
    cnt = torch.where(cnt == 0, torch.tensor(1), cnt)
    assert (cnt > 1).any() and (cnt == 1).any()
    assert torch.equal(got.to(dt), buf / cnt)            # demofusion.py:259-264, both operands in the latent dtype


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("mixture", [True, False])
def test_emulated_offset_combine_equals_eager(emul, dn, mixture):
    dt = DTYPES[dn]
    N, C, H, W, s, off = 2, 4, 60, 76, 2, 6
    end = W - off
    end_y, end_x = min(H, end), end
    oh, ow = len(range(off, end_y, s)), len(range(off, end_x, s))
    views = [(0, 0), (1, 0), (0, 1), (1, 1)] * (2 if mixture else 1)
    nv = len(views)
    outv = synth.latent(21, (nv * N, C, oh, ow), dt)
    x_local = synth.latent(22, (N, C, H, W), dt)
    res = torch.empty_like(x_local)
    vpb = 3                                              # deliberately not a divisor of the view count
    nbat = -(-nv // vpb)
    batches = [outv[b * vpb * N:min((b + 1) * vpb, nv) * N].contiguous() for b in range(nbat)]
    ptrs = (ctypes.c_void_p * nbat)(*[b.data_ptr() for b in batches])
    c2 = 0.3125
    emul.td_emul_combine_offset(_p(x_local), ptrs, nbat, vpb, nv, _p(res), N, C, H, W, s, oh, ow, off, end_y, end_x, int(mixture),
                                ctypes.c_float(c2), ctypes.c_float(1 - c2), CODE[dt])
    xg = torch.zeros_like(x_local)
    for idx, (bx, by) in enumerate(views):
        xg[:, :, by + off:end:s, bx + off:end:s] += outv[idx * N:(idx + 1) * N]
    if mixture:
        xg = xg / 2
    want = x_local * (1 - c2) + xg * c2
    assert torch.equal(res, want)


@pytest.mark.parametrize("dn,mixture", [("f32", True), ("f16", False)])
def test_delegate_jitter_step_on_emulated_kernels_matches_reference_fixture(emul, monkeypatch, golden_dir, dn, mixture):
    """The whole DemoFusion jitter step of OUR delegate with the three td_jitter.cu kernels replaced by their host
    emulation (everything else on torch stand-ins), against the fixture generated from the unmodified reference."""
    from helpers import install_demofusion_stand_ins
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from oracle import demofusion as odf
    from oracle.make_golden import DEMO_CFG, position_aware_denoise
    from test_demofusion import _jitter_delegate, _jitter_oracle
    install_demofusion_stand_ins(monkeypatch.setattr)

    def origins_np(origins_dev):
        return np.ascontiguousarray(origins_dev.numpy().astype(np.int32))

    def scatter_bboxes(x, origins_dev, origins_host, n_tiles, tile_h, tile_w, out=None):
        N, C, H, W = x.shape
        x = x.contiguous()
        tiles = torch.empty((n_tiles * N, C, tile_h, tile_w), dtype=x.dtype)
        o = origins_np(origins_dev)
        emul.td_emul_scatter_bboxes(_p(x), _p(tiles), o.ctypes.data_as(ctypes.c_void_p), n_tiles, N, C, H, W, tile_h, tile_w, x.element_size())
        return tiles

    def blend_bboxes(batch_outs, tile_bs, origins_dev, origins_host, n_tiles, N, C, H, W, tile_h, tile_w):
        keep = [t.contiguous() for t in batch_outs]
        ptrs = (ctypes.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
        out = torch.empty((N, C, H, W), dtype=torch.float32)
        o = origins_np(origins_dev)
        emul.td_emul_blend_bboxes(ptrs, len(keep), tile_bs, o.ctypes.data_as(ctypes.c_void_p), n_tiles, N, C, H, W, tile_h, tile_w,
                                  CODE[keep[0].dtype], _p(out))
        return out

    def demofusion_combine(x_local, view_outs, views_per_batch, n_views, s, out_h, out_w, offset, end_y, end_x, mixture, c2, one_minus_c2):
        N, C, H, W = x_local.shape
        keep = [t.contiguous() for t in view_outs]
        ptrs = (ctypes.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
        out = torch.empty_like(x_local)
        emul.td_emul_combine_offset(_p(x_local.contiguous()), ptrs, len(keep), views_per_batch, n_views, _p(out), N, C, H, W, s, out_h, out_w,
                                    offset, end_y, end_x, int(mixture), ctypes.c_float(c2), ctypes.c_float(one_minus_c2), CODE[x_local.dtype])
        return out
    monkeypatch.setattr(engine, "scatter_bboxes", scatter_bboxes)
    monkeypatch.setattr(engine, "blend_bboxes", blend_bboxes)
    monkeypatch.setattr(engine, "demofusion_combine", demofusion_combine)

    c = DEMO_CFG
    name = f"{dn}_{'mixture' if mixture else 'plain'}_jitter"
    g = np.load(os.path.join(golden_dir, "demofusion_jitter.npz"))
    x, xp, _, local, sizes = _jitter_oracle(DTYPES[dn], mixture)
    d = _jitter_delegate(mixture)
    d.sampler_forward = position_aware_denoise(d)
    d.cosine_factor = odf.cosine_factor(c["current_step"], c["t_enc"])
    cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8)], "c_concat": [torch.zeros(c["N"], 5, 1, 1)]}
    got = d.sample_one_step(xp, torch.ones(c["N"]), cond)
    want = torch.from_numpy(g[name].view(np.float32 if dn == "f32" else np.float16).copy())
    tol = 3e-6 if dn == "f32" else 2e-3
    err = (got.float() - want.float()).abs().max().item()
    assert got.shape == want.shape and err <= tol * max(1.0, want.float().abs().max().item()), f"max err {err}"
