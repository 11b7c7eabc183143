"""Seamless DemoFusion on the GPU: td_depthwise_conv2d_wrap against a float64 circular convolution, the wrap list scatter
and blend bit for bit against tests/demofusion_wrap_oracle.py, the delegate's step against its demofusion_step (small
canvases at every scale and one cfg5-size canvas), the seam property, and the wrapped delegate on a one-rank NCCL group."""
import ctypes
import os
import random
import socket
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import demofusion_wrap_oracle as dwo
import wrap_oracle as wo
from oracle import demofusion as odf
from oracle import synth
from oracle.make_golden import demo_denoise
from test_demofusion_wrap import WRAPS, oracle_list_blend, ring_windows, windows_of
from test_gpu_demofusion_kernels import CS2, CS3, DTS, OVERLAP, SEED, SIG, TILE_BS, WINDOW, _conv, _conv_violations, _latent, _step_size

pytestmark = pytest.mark.gpu


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def _conv_wrap(x, taps, wrap):
    cabi = _cabi()
    out = torch.empty_like(x)
    w = np.ascontiguousarray(taps.float().numpy())
    cabi.check(cabi.lib.td_depthwise_conv2d_wrap(x.data_ptr(), out.data_ptr(), x.shape[0] * x.shape[1], x.shape[2], x.shape[3],
                                                 w.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), taps.shape[0], wrap,
                                                 cabi.dtype_code(x.dtype), cabi.current_stream_ptr()))
    return out


def _conv64_wrap(x, taps, wrap):
    """Depthwise conv in float64 on the host, circular on the wrapped axes, zero padding on the others: (value, sum |x*w|)."""
    C, k = x.shape[1], taps.shape[0]
    r = k // 2
    w = taps.double()[None, None].repeat(C, 1, 1, 1)
    px, py = (r if wrap & wo.WRAP_X else 0), (r if wrap & wo.WRAP_Y else 0)
    pad = (0 if wrap & wo.WRAP_Y else r, 0 if wrap & wo.WRAP_X else r)
    xd = F.pad(x.cpu().double(), (px, px, py, py), mode="circular")
    return F.conv2d(xd, w, padding=pad, groups=C), F.conv2d(xd.abs(), w.abs(), padding=pad, groups=C)


@pytest.mark.parametrize("wn", list(WRAPS))
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("s", [1, 3, 5, 8])
def test_wrap_conv_against_float64(s, dn, wn):
    """The class's gaussian and a random asymmetric kernel, on an odd canvas and on one whose wrapped axes are as short as the
    kernel radius allows (k/2 == L: every tap wraps); the rounding bound of test_depthwise_conv_against_float64.  wrap = 0
    is bit-equal to td_depthwise_conv2d."""
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    dt, k, wrap = DTS[dn], 2 * s - 1, WRAPS[wn]
    sigma = 0.6 * float(0.99 * odf.cosine_factor(3, 14) + 1e-2)
    gauss = DemoFusion.gaussian_kernel(None, k, sigma, 1)[0, 0].to(dt).float()
    g = torch.Generator().manual_seed(s)
    asym = torch.rand((k, k), generator=g, dtype=torch.float64) - 0.3
    asym = (asym / asym.abs().sum()).to(dt).float()
    r = max(1, k // 2)
    shapes = [(2, 4, 37, 53), (1, 2, r if wrap & wo.WRAP_Y else 5, r if wrap & wo.WRAP_X else 6)]
    for taps, name in ((gauss, "gaussian"), (asym, "asymmetric")):
        for si, shape in enumerate(shapes):
            x = _latent(700 + 10 * s + si, shape, dt).cuda()
            got = _conv_wrap(x, taps, wrap)
            ref, absref = _conv64_wrap(x, taps, wrap)
            assert _conv_violations(got, ref, absref, k, dt) == 0, f"k {k} {name} {shape} {dt} wrap {wrap}"
            if name == "asymmetric" and k > 1 and si == 0:
                assert _conv_violations(_conv_wrap(x, taps.flip(0, 1), wrap), ref, absref, k, dt) > 0
                assert _conv_violations(_conv(x, taps), ref, absref, k, dt) > 0, "the zero-padded conv must miss the seam"
            assert torch.equal(_conv_wrap(x, taps, 0), _conv(x, taps))


@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("wn", ["none", "x", "y", "xy"])
def test_wrap_list_scatter_and_blend_are_bit_exact(dn, wn):
    """128 windows in 128 batch tensors (the pointer-table limit), across the seams and off the bounded edges; signed zeros
    in the latent and the tile outputs must come back as the oracle has them."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    dt, wrap = DTS[dn], WRAPS.get(wn, 0)
    N, C, H, W, ws, T = 2, 4, 64, 96, 16, 128
    windows = ring_windows(T, H, W, ws, ws, wrap, 11 + wrap)
    flat = [v for b in windows for v in b[:2]]
    host = (ctypes.c_int32 * len(flat))(*flat)
    dev = torch.tensor(flat, dtype=torch.int32, device="cuda")
    x = synth.latent(61, (N, C, H, W), dt)
    x[:, :, ::7, ::5] = -0.0
    xd = x.cuda()
    if wrap:
        tiles = engine.scatter_bboxes(xd, dev, host, T, ws, ws, wrap=wrap)
    else:   # wrap = 0: the same list form with both axes bounded (negative origins, which td_scatter_bboxes refuses)
        tiles = torch.empty((T * N, C, ws, ws), dtype=dt, device="cuda")
        _cabi().check(_cabi().lib.td_scatter_bboxes_wrap(xd.data_ptr(), tiles.data_ptr(), dev.data_ptr(), host, T, N, C, H, W, ws, ws, 0,
                                                         _cabi().dtype_code(dt), _cabi().current_stream_ptr()))
    want = torch.cat([dwo.demofusion_crop(x, b, wrap) for b in windows], dim=0)
    iv = torch.int32 if dt == torch.float32 else torch.int16
    assert torch.equal(tiles.cpu().view(iv), want.view(iv))

    outs_all = synth.latent(62, (T * N, C, ws, ws), dt)
    outs_all[::3, :, ::2] = -0.0
    outs = [outs_all[t * N:(t + 1) * N].cuda() for t in range(T)]
    ptrs = (ctypes.c_void_p * T)(*[o.data_ptr() for o in outs])
    got = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")
    _cabi().check(_cabi().lib.td_blend_bboxes_wrap(ptrs, T, 1, dev.data_ptr(), host, T, N, C, H, W, ws, ws, wrap, _cabi().dtype_code(dt),
                                                   got.data_ptr(), _cabi().current_stream_ptr()))
    want = oracle_list_blend(outs_all, windows, N, (N, C, H, W), dt, wrap)
    g = got.cpu().to(dt)
    assert torch.equal(g.view(iv), want.view(iv))


def _wrap_delegate(s, mixture, jitter, h, w, tile_bs_g, wrap):
    from test_gpu_demofusion_kernels import _delegate
    d = _delegate(s, mixture, jitter, h, w, tile_bs_g)
    random.seed(SEED)
    d.get_views(OVERLAP, TILE_BS, tile_bs_g, wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    return d


STEP_CASES = [(s, kind, jitter) for s in (1, 3, 5, 8) for kind in ("landscape", "portrait") for jitter in (False, True)]


@pytest.mark.parametrize("wn", list(WRAPS))
@pytest.mark.parametrize("dn", list(DTS))
@pytest.mark.parametrize("mixture", [False, True], ids=["plain", "mixture"])
@pytest.mark.parametrize("s,kind,jitter", STEP_CASES, ids=[f"s{s}-{k}-{'jitter' if j else 'grid'}" for s, k, j in STEP_CASES])
def test_wrapped_sample_one_step_matches_oracle(s, kind, jitter, mixture, dn, wn):
    """The axes of test_sample_one_step_matches_oracle on a seamless canvas: the latent is not padded, the output has its
    shape, and the step equals demofusion_wrap_oracle.demofusion_step with that test's tolerances."""
    dt, wrap = DTS[dn], WRAPS[wn]
    h, w, _ = _step_size(s, kind, False)
    tile_bs_g = 1 if s == 8 else 3
    d = _wrap_delegate(s, mixture, jitter, h, w, tile_bs_g, wrap)
    local, jr = dwo.demofusion_views(w, h, WINDOW, OVERLAP, wrap, random.Random(SEED) if jitter else None)
    assert windows_of(d) == local and d.jitter_range == jr
    N, C = 2, 4
    x = synth.latent(900 + s, (N, C, h, w), dt)
    lb = [local[i * d.tile_bs:(i + 1) * d.tile_bs] for i in range(d.num_batches)]
    views = odf.global_views(s, mixture)
    gb = [views[i * d.global_tile_bs:(i + 1) * d.global_tile_bs] for i in range(d.global_num_batches)]
    want = dwo.demofusion_step(x, lb, gb, s, mixture, True, SIG, d.cosine_factor, CS2, CS3, lambda t, b: synth.fake_denoise(t, b, N),
                               lambda t, b: demo_denoise(t), wrap=wrap, jitter_range=jr)
    cond = {"c_crossattn": [torch.zeros(N, 77, 8, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
    got = d.sample_one_step(x.cuda(), torch.ones(N, device="cuda"), cond)
    assert got.dtype == dt and got.shape == want.shape == x.shape
    tol = {torch.float32: 3e-6, torch.float16: 2e-3, torch.bfloat16: 1.6e-2}[dt]
    err = (got.cpu().float() - want.float()).abs().max().item()
    assert err <= tol * max(1.0, want.float().abs().max().item()), f"{h}x{w} wrap {wrap}: max err {err}"


@pytest.mark.parametrize("jitter", [False, True], ids=["grid", "jitter"])
def test_wrapped_cfg5_size_step_matches_oracle(jitter):
    """cfg5's geometry (latent [2,4,768,768] fp16, window 128, stride 64, scale 4, mixture) wrapped on both axes: 12 x 12 =
    144 ring windows, against the oracle on the host."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    c = bench.DEMO
    wrap = wo.WRAP_X | wo.WRAP_Y
    d, _, _ = bench._demo_job(torch.device("cuda"), torch.float16, True, jitter)
    random.seed(SEED)
    d.get_views(c["overlap"], c["tile_bs"], c["tile_bs_g"], wrap_x=True, wrap_y=True)
    d.sampler_forward = lambda x_tile, sigma=None, cond=None: demo_denoise(x_tile)
    cf = odf.cosine_factor(c["current_step"], c["t_enc"])
    d.cosine_factor = cf
    L = c["lat"]
    local, jr = dwo.demofusion_views(L, L, c["window"], c["overlap"], wrap, random.Random(SEED) if jitter else None)
    assert windows_of(d) == local and len(local) == 144
    x = synth.latent(77, (c["N"], c["C"], L, L), torch.float16)
    lb = [local[i * d.tile_bs:(i + 1) * d.tile_bs] for i in range(d.num_batches)]
    views = odf.global_views(c["scale"], True)
    gb = [views[i * d.global_tile_bs:(i + 1) * d.global_tile_bs] for i in range(d.global_num_batches)]
    want = dwo.demofusion_step(x, lb, gb, c["scale"], True, True, c["sig"], cf, c["cs2"], c["cs3"], lambda t, b: demo_denoise(t),
                               lambda t, b: demo_denoise(t), wrap=wrap, jitter_range=jr)
    cond = {"c_crossattn": [torch.zeros(c["N"], 77, 8, device="cuda")], "c_concat": [torch.zeros(c["N"], 5, 1, 1, device="cuda")]}
    got = d.sample_one_step(x.cuda(), torch.ones(c["N"], device="cuda"), cond)
    assert got.dtype == torch.float16 and got.shape == want.shape
    err = (got.cpu().float() - want.float()).abs().max().item()
    assert err <= 2e-3 * max(1.0, want.float().abs().max().item()), f"max err {err}"


def test_step_commutes_with_a_roll():
    """The seam property, as for MultiDiffusion in test_gpu_wrap.py.  A wrap-xy canvas L = 256, window 64, overlap 32
    (stride 32, a multiple of s = 2, dividing L) and a position-independent stand-in (tile-local blur, views x 0.5):
    rolling the latent by one stride and stepping equals stepping and rolling, up to the summation order of the statistics
    and of the blend at the seam (fp32: 1e-6 relative).  The bounded delegate fails the same check at the edges."""
    from test_gpu_demofusion_kernels import _delegate
    N, C, L, s = 1, 4, 256, 2
    x = torch.randn((N, C, L, L), generator=torch.Generator().manual_seed(5)).cuda()
    cond = {"c_crossattn": [torch.zeros(N, 77, 8, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}

    def step(wrap, xx):
        d = _delegate(s, True, False, L, L, 3)
        d.window_size = 64
        d.get_views(32, TILE_BS, 3, wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
        d.sampler_forward = lambda xt, sigma=None, cond=None: wo.blur_denoise(xt) if xt.shape[-1] == 64 else demo_denoise(xt)   # views: 128
        assert d.stride == 32
        return d.sample_one_step(xx, torch.ones(N, device="cuda"), cond)
    for wrap, must_hold in ((wo.WRAP_X | wo.WRAP_Y, True), (0, False)):
        a = torch.roll(step(wrap, x), (32, 32), (2, 3))
        b = step(wrap, torch.roll(x, (32, 32), (2, 3)))
        rel = ((a - b).abs().max() / b.abs().max()).item()
        assert (rel <= 1e-6) == must_hold, f"wrap {wrap}: relative difference {rel}"


def test_wrapped_delegate_on_a_one_rank_nccl_group_is_bit_identical():
    import torch.distributed as dist
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        h, w, _ = _step_size(3, "landscape", False)
        N, C = 2, 4
        x = synth.latent(11, (N, C, h, w), torch.float16).cuda()
        cond = {"c_crossattn": [torch.zeros(N, 77, 8, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
        for jitter in (False, True):
            for wrap in WRAPS.values():
                single = _wrap_delegate(3, True, jitter, h, w, 3, wrap).sample_one_step(x, torch.ones(N, device="cuda"), cond)
                d = _wrap_delegate(3, True, jitter, h, w, 3, wrap)
                d.init_tile_shard(None)
                sharded = d.sample_one_step(x, torch.ones(N, device="cuda"), cond)
                assert torch.equal(sharded.view(torch.int16), single.view(torch.int16)), f"jitter {jitter} wrap {wrap}"
    finally:
        dist.destroy_process_group()
