"""GPU tests of everything written after the round-1 GPU budget was spent: region prompt control, ControlNet tile caches,
DemoFusion random jitter (the list-driven kernels of csrc/td_jitter.cu).  Their host logic is pinned on CPU against the
reference (tests/test_region*.py, test_side_inputs.py, test_demofusion.py); the device runs below have not executed on
hardware when they were written; they are plain tests now.

The file sorts last on purpose: should a never-run kernel fault, the CUDA context of the pytest process is gone, and
nothing that is already verified may run after it.
"""
import os
import types

import numpy as np
import pytest
import torch

from helpers import load_golden, DTYPES, assert_bit_equal
from oracle import demofusion as odf
from oracle import synth
from oracle.make_golden import DEMO_CFG, REGION_CASES, REGION_DTYPES
from test_demofusion import _jitter_delegate, _jitter_oracle
from test_region import _run_delegate, _want, _x
from test_side_inputs import H, W, _hints, _p


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "region_small")


# ------------------------------------------------------------------------------- region prompt control (verified kernels + torch)
@pytest.mark.gpu
@pytest.mark.parametrize("case", REGION_CASES, ids=[c[0] for c in REGION_CASES])
@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", REGION_DTYPES)
def test_delegate_region_step_on_gpu(gold, case, method, dn):
    name, bg, rows = case
    d, out = _run_delegate(method, _x(name, dn), bg, rows, "cuda")
    assert out.is_cuda
    assert_bit_equal(out, _want(gold, f"{name}_{method}_{dn}"), f"{method} delegate, sm_90a kernels")


# ------------------------------------------------------------------------------- ControlNet tile caches (scatter on the x8 plan)
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_controlnet_tile_caches_on_gpu_equal_plain_slicing(dtype):
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion

    class _K:
        model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None, step=0)
    d = MultiDiffusion(_p(), _K())
    d.init_grid_bbox(16, 16, 8, 4)
    hints = [t.to(dtype) for t in _hints("cuda")]
    want_src = [t.clone() if t.dim() == 4 else t.clone().unsqueeze(0) for t in hints]
    cs = types.SimpleNamespace(latest_network=types.SimpleNamespace(control_params=[types.SimpleNamespace(hint_cond=t) for t in hints]))
    d.init_controlnet(cs, False)
    d.init_done()
    for pid, src in enumerate(want_src):
        for b, bboxes in enumerate(d.batched_bboxes):
            want = torch.cat([src[:, :, bb[1] * 8:bb[3] * 8, bb[0] * 8:bb[2] * 8] for bb in bboxes], dim=0)
            got = d.control_tensor_batch[pid][b]
            assert got.is_cuda and got.shape == want.shape and torch.equal(got, want)
    d.switch_controlnet_tensors(1, 2, len(d.batched_bboxes[1]))
    got = cs.latest_network.control_params[0].hint_cond
    want = torch.cat([want_src[0][:, :, bb[1] * 8:bb[3] * 8, bb[0] * 8:bb[2] * 8].repeat(2, 1, 1, 1) for bb in d.batched_bboxes[1]], dim=0)
    assert torch.equal(got, want)
    d.reset_controlnet_tensors()
    assert cs.latest_network.control_params[0].hint_cond.shape == (1, 3, H * 8, W * 8)


# ------------------------------------------------------------------------------- strip form of the MultiDiffusion blend (new kernel)
STRIP = 128


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("use_rcp", [False, True])
@pytest.mark.parametrize("STRIP", [128, 128 | 64], ids=["two_planes", "one_plane"])
def test_strip_blend_matches_reference_fixtures_on_gpu(golden_dir, dn, use_rcp, STRIP):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from helpers import bits, sha
    from test_gpu_diffusion import _run_cuda_step
    if use_rcp and dn == "f32":
        pytest.skip("the fast exact divide is a 16-bit path")
    g = load_golden(golden_dir, "blend_small")
    for name, (N, C, W, H, tw, th, ov, bs) in zip(g["names"], g["cases"]):
        x = synth.latent(synth.case_seed(str(name), dn), (int(N), int(C), int(H), int(W)), DTYPES[dn])
        out, xb, plan = _run_cuda_step(engine, "md", x, int(W), int(H), int(tw), int(th), int(ov), int(bs), flags=STRIP, use_rcp=use_rcp)
        assert np.array_equal(bits(out), g[f"{name}_{dn}_md"]), f"{name}: strip blend differs from the reference's"
    if dn == "f16":
        h = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
        idx = list(h["names"]).index("cfg2_ov48")
        N, C, W, H, tw, th, ov, bs = (int(v) for v in h["cases"][idx])
        x = synth.latent(synth.case_seed("cfg2_ov48", dn), (N, C, H, W), DTYPES[dn])
        out, _, _ = _run_cuda_step(engine, "md", x, W, H, tw, th, ov, bs, flags=STRIP, use_rcp=use_rcp)
        assert sha(out) == str(h["cfg2_ov48_f16_md"])


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_strip_mixture_matches_reference_fixtures_on_gpu(golden_dir, dn):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from helpers import bits, sha
    from test_gpu_diffusion import _run_cuda_step
    g = load_golden(golden_dir, "blend_small")
    for name, (N, C, W, H, tw, th, ov, bs) in zip(g["names"], g["cases"]):
        x = synth.latent(synth.case_seed(str(name), dn), (int(N), int(C), int(H), int(W)), DTYPES[dn])
        out, _, _ = _run_cuda_step(engine, "mod", x, int(W), int(H), int(tw), int(th), int(ov), int(bs), flags=STRIP)
        assert np.array_equal(bits(out), g[f"{name}_{dn}_mod"]), f"{name}: strip Mixture of Diffusers differs from the reference's"
    if dn == "f16":
        h = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
        idx = list(h["names"]).index("cfg2_ov48")
        N, C, W, H, tw, th, ov, bs = (int(v) for v in h["cases"][idx])
        x = synth.latent(synth.case_seed("cfg2_ov48", dn), (N, C, H, W), DTYPES[dn])
        out, _, _ = _run_cuda_step(engine, "mod", x, W, H, tw, th, ov, bs, flags=STRIP)
        assert sha(out) == str(h["cfg2_ov48_f16_mod"])


# ------------------------------------------------------------------------------- DemoFusion random jitter (new kernels: last)
@pytest.mark.gpu
@pytest.mark.parametrize("dn,mixture", [("f32", True), ("f16", False), ("f16", True)])
def test_demofusion_jitter_class_matches_oracle(dn, mixture):
    from oracle.make_golden import position_aware_denoise
    c = DEMO_CFG
    x, xp, want, local, sizes = _jitter_oracle(DTYPES[dn], mixture)
    d = _jitter_delegate(mixture)
    assert [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb] == local
    d.sampler_forward = position_aware_denoise(d)
    d.cosine_factor = odf.cosine_factor(c["current_step"], c["t_enc"])
    cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8, device="cuda")], "c_concat": [torch.zeros(c["N"], 5, 1, 1, device="cuda")]}
    got = d.sample_one_step(xp.cuda(), torch.ones(c["N"], device="cuda"), cond)
    assert got.dtype == DTYPES[dn] and got.shape == want.shape
    tol = 3e-6 if dn == "f32" else 2e-3
    err = (got.cpu().float() - want.float()).abs().max().item()
    assert err <= tol * max(1.0, want.float().abs().max().item()), f"max err {err}"
    # get_noise pads and crops around the same step (demofusion.py:345-353)
    d.p.sd_model = types.SimpleNamespace(apply_model=lambda xt, s_, cond=None: d.sampler_forward(xt, s_, cond=cond))
    d.t_enc = c["t_enc"]
    eps = d.get_noise(x.cuda(), torch.ones(c["N"], device="cuda"), cond, 0)
    jr = d.jitter_range
    err = (eps.cpu().float() - want[:, :, jr:jr + c["H"], jr:jr + c["W"]].float()).abs().max().item()
    assert eps.shape == x.shape and err <= tol * max(1.0, want.float().abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_window_list_scatter_and_blend_are_exact(dn):
    """td_scatter_bboxes == slicing + cat; td_blend_bboxes == the eager per-window add / count / divide, bit for bit."""
    import ctypes
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import check, current_stream_ptr, dtype_code, lib
    dt = DTYPES[dn]
    N, C, H, W, ws, tile_bs = 2, 3, 45, 70, 16, 4
    rng = np.random.default_rng(11)
    T = 13
    org = [(int(rng.integers(0, W - ws + 1)), int(rng.integers(0, H - ws + 1))) for _ in range(T)]
    flat = [v for o in org for v in o]
    host_arr = (ctypes.c_int32 * len(flat))(*flat)
    dev_arr = torch.tensor(flat, dtype=torch.int32, device="cuda")
    x = synth.latent(12, (N, C, H, W), dt).cuda()
    tiles = torch.empty((T * N, C, ws, ws), dtype=dt, device="cuda")
    check(lib.td_scatter_bboxes(x.data_ptr(), tiles.data_ptr(), dev_arr.data_ptr(), host_arr, T, N, C, H, W, ws, ws, dtype_code(dt),
                                current_stream_ptr()))
    assert torch.equal(tiles, torch.cat([x[:, :, oy:oy + ws, ox:ox + ws] for ox, oy in org], dim=0))
    outs_src = synth.latent(13, (T * N, C, ws, ws), dt).cuda()
    nb = -(-T // tile_bs)
    outs = [outs_src[b * tile_bs * N:min((b + 1) * tile_bs, T) * N].contiguous() for b in range(nb)]
    ptrs = (ctypes.c_void_p * nb)(*[o.data_ptr() for o in outs])
    got = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")
    check(lib.td_blend_bboxes(ptrs, nb, tile_bs, dev_arr.data_ptr(), host_arr, T, N, C, H, W, ws, ws, dtype_code(dt), got.data_ptr(),
                              current_stream_ptr()))
    buf = torch.zeros_like(x)
    cnt = torch.zeros_like(x)
    for t, (ox, oy) in enumerate(org):
        buf[:, :, oy:oy + ws, ox:ox + ws] += outs_src[t * N:(t + 1) * N]
        cnt[:, :, oy:oy + ws, ox:ox + ws] += 1
    cnt = torch.where(cnt == 0, torch.tensor(1, device="cuda"), cnt)
    want = buf / cnt
    assert torch.equal(got.to(dt), want)
    # a window that leaves the canvas is refused with a status, not a fault
    bad = (ctypes.c_int32 * 2)(W - ws + 1, 0)
    assert lib.td_scatter_bboxes(x.data_ptr(), tiles.data_ptr(), dev_arr.data_ptr(), bad, 1, N, C, H, W, ws, ws, dtype_code(dt),
                                 current_stream_ptr()) < 0


@pytest.mark.gpu
def test_combine_with_offset_is_exact():
    import ctypes
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import check, current_stream_ptr, lib
    N, C, H, W, s, off = 2, 4, 60, 76, 2, 6
    end = W - off
    end_y, end_x = min(H, end), end
    oh, ow = len(range(off, end_y, s)), len(range(off, end_x, s))
    views = [(0, 0), (1, 0), (0, 1), (1, 1)] * 2
    outv = synth.latent(21, (8 * N, C, oh, ow), torch.float16).cuda()
    x_local = synth.latent(22, (N, C, H, W), torch.float16).cuda()
    res = torch.empty_like(x_local)
    ptrs = (ctypes.c_void_p * 2)(outv[:4 * N].data_ptr(), outv[4 * N:].data_ptr())
    c2 = 0.3125
    check(lib.td_demofusion_combine_offset(x_local.data_ptr(), ptrs, 2, 4, 8, res.data_ptr(), N, C, H, W, s, oh, ow, off, end_y, end_x, 1,
                                           c2, 1 - c2, 0, current_stream_ptr()))
    xg = torch.zeros_like(x_local)
    for idx, (bx, by) in enumerate(views):
        xg[:, :, by + off:end:s, bx + off:end:s] += outv[idx * N:(idx + 1) * N]
    want = x_local * (1 - c2) + (xg / 2) * c2
    assert torch.equal(res, want)
