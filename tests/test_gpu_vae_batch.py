"""Batched tensor-core VAE pass: N images through the tiles together, each with its own GroupNorm statistics.

The acceptance bar is bit-equality with the one-image schedule: every batched kernel is compared with its one-image
form image by image, and VAEHook with several images per pass with `images_per_pass = 1`."""
import ctypes
import json
import os
import tempfile

import pytest
import torch

from helpers import assert_bit_equal

pytestmark = pytest.mark.gpu

DTS = {"f16": torch.float16, "bf16": torch.bfloat16}
NS = (1, 2, 3, 8)


@pytest.fixture(scope="module")
def m():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, host, tilevae, vae_engine, vae_ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _cabi, vae_ops, vae_engine, tilevae, host


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _per_image_scaled(shape, dtype, seed):
    """Images that differ by orders of magnitude: a statistic taken from the wrong image shows."""
    x = _rand(shape, dtype, seed)
    for n in range(shape[0]):
        x[n] = (x[n].float() * 10.0 ** (n % 3 - 1) + n).to(dtype)
    return x


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------ GroupNorm statistics / apply
def _stats_one(cabi, x1, C, groups):
    """td_gn_stats_nhwc of one image [pixels, C] -> (mean, var)."""
    P = x1.numel() // C
    ws_bytes = cabi.lib.td_gn_stats_nhwc_workspace_bytes(P, C, groups)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    mean = torch.empty(groups, dtype=torch.float32, device="cuda")
    var = torch.empty(groups, dtype=torch.float32, device="cuda")
    cabi.check(cabi.lib.td_gn_stats_nhwc(x1.data_ptr(), P, C, groups, cabi.dtype_code(x1.dtype), ws.data_ptr(), ws_bytes,
                                         mean.data_ptr(), var.data_ptr(), cabi.current_stream_ptr()))
    return mean, var


def _apply_one(cabi, x1, C, groups, mean, var, gamma, beta, act, out=None):
    P = x1.numel() // C
    y = torch.empty_like(x1) if out is None else out
    cabi.check(cabi.lib.td_gn_apply_nhwc(x1.data_ptr(), y.data_ptr(), P, C, groups, cabi.dtype_code(x1.dtype), mean.data_ptr(),
                                         var.data_ptr(), gamma.data_ptr() if gamma is not None else None,
                                         beta.data_ptr() if beta is not None else None, 1e-6, int(act), cabi.current_stream_ptr()))
    return y


def _pixel_cases(C):
    """Odd counts, fewer pixels than one CTA iteration covers, and both sides of where the statistics grid saturates
    (ceil(P / ppi) == 4 * SMs)."""
    ppi = 256 // (C // 8)
    sat = ppi * 4 * _sms()
    return sorted({1, 3, max(ppi - 1, 1), ppi + 1, 1237, sat - 1, sat + 1})


@pytest.mark.parametrize("C", [128, 256, 512])
@pytest.mark.parametrize("dt", list(DTS))
def test_batched_stats_and_apply_are_the_one_image_bits(m, dt, C):
    cabi, ops, *_ = m
    dtype = DTS[dt]
    groups = 32
    for N in NS:
        for P in _pixel_cases(C):
            x = _per_image_scaled((N, 1, P, C), dtype, seed=N * 7919 + P + C)
            var, mean = ops.gn_stats_nhwc(x, groups)
            gamma = _rand((C,), torch.float32, 3) + 1.0
            beta = _rand((C,), torch.float32, 4)
            for act in (False, True):
                y = ops.gn_apply_nhwc(x, mean, var, gamma if act else None, beta if act else None, act)
                for n in range(N):
                    want_mean, want_var = _stats_one(cabi, x[n], C, groups)
                    sl = slice(n * groups, (n + 1) * groups)
                    assert_bit_equal(mean[sl], want_mean, f"{dt} C={C} N={N} P={P} mean of image {n}")
                    assert_bit_equal(var[sl], want_var, f"{dt} C={C} N={N} P={P} var of image {n}")
                    want = _apply_one(cabi, x[n], C, groups, want_mean, want_var, gamma if act else None, beta if act else None, act)
                    assert_bit_equal(y[n], want, f"{dt} C={C} N={N} P={P} act={act} apply of image {n}")
            inplace = x.clone()
            ops.gn_apply_nhwc(inplace, mean, var, None, None, False, inplace=True)
            assert_bit_equal(inplace, ops.gn_apply_nhwc(x, mean, var, None, None, False), f"{dt} C={C} N={N} P={P} in place")


def test_batched_stats_and_apply_past_2_31_elements(m):
    """N * pixels * C = 2^31 + 3072: the second image starts past 2^31 elements (2^32 bytes)."""
    cabi, ops, *_ = m
    C, P = 512, (1 << 21) + 3
    x = torch.empty((2, 1, P, C), dtype=torch.float16, device="cuda")
    x[0].copy_(_rand((1, P, C), torch.float16, 11))
    x[1].copy_(_rand((1, P, C), torch.float16, 12, scale=50.0) + 7)
    assert x.numel() > 1 << 31
    var, mean = ops.gn_stats_nhwc(x)
    for n in range(2):
        want_mean, want_var = _stats_one(cabi, x[n], C, 32)
        assert_bit_equal(mean[n * 32:(n + 1) * 32], want_mean, f"mean of image {n}")
        assert_bit_equal(var[n * 32:(n + 1) * 32], want_var, f"var of image {n}")
    want_last = _apply_one(cabi, x[1], C, 32, mean[32:], var[32:], None, None, True)
    ops.gn_apply_nhwc(x, mean, var, None, None, True, inplace=True)
    assert_bit_equal(x[1], want_last, "apply of the image past 2^31")
    del x, want_last
    torch.cuda.empty_cache()


def test_batched_norm_entries_refuse_and_leave_outputs_untouched(m):
    cabi, ops, *_ = m
    lib, C, P, N = cabi.lib, 128, 37, 2
    x = _rand((N * P * C + 8,), torch.float16, 5)
    ws_bytes = lib.td_gn_stats_nhwc_batched_workspace_bytes(N, P, C, 32)
    assert ws_bytes == N * lib.td_gn_stats_nhwc_workspace_bytes(P, C, 32)
    assert lib.td_gn_stats_nhwc_batched_workspace_bytes(0, P, C, 32) == 0
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    mean = torch.full((N * 32,), 7.0, device="cuda")
    var = torch.full((N * 32,), 7.0, device="cuda")
    y = torch.full((N * P * C,), 3.0, dtype=torch.float16, device="cuda")
    s, f16 = cabi.current_stream_ptr(), cabi.TD_F16
    need = N * -(-P // (256 // (C // 8))) * 32 * 3 * 4      # N images x the one-image grid x groups x (n, mean, M2)
    stats = lambda xp=x.data_ptr(), n=N, p=P, c=C, g=32, wb=ws_bytes: lib.td_gn_stats_nhwc_batched(xp, n, p, c, g, f16, ws.data_ptr(), wb, mean.data_ptr(), var.data_ptr(), s)
    apply = lambda xp=x.data_ptr(), yp=y.data_ptr(), n=N, p=P, c=C, g=32: lib.td_gn_apply_nhwc_batched(xp, yp, n, p, c, g, f16, mean.data_ptr(), var.data_ptr(), None, None, 1e-6, 1, s)
    cases = [
        (stats(n=0), cabi.TD_ERR_INVALID_ARG), (stats(n=65536), cabi.TD_ERR_INVALID_ARG), (stats(p=0), cabi.TD_ERR_INVALID_ARG),
        (stats(xp=x.data_ptr() + 2), cabi.TD_ERR_INVALID_ARG), (stats(c=120), cabi.TD_ERR_UNSUPPORTED), (stats(g=3), cabi.TD_ERR_UNSUPPORTED),
        (stats(wb=need - 4), cabi.TD_ERR_CAPACITY), (stats(xp=None), cabi.TD_ERR_INVALID_ARG),
        (apply(n=0), cabi.TD_ERR_INVALID_ARG), (apply(n=65536), cabi.TD_ERR_INVALID_ARG), (apply(xp=x.data_ptr() + 2), cabi.TD_ERR_INVALID_ARG),
        (apply(yp=y.data_ptr() + 2), cabi.TD_ERR_INVALID_ARG), (apply(c=120), cabi.TD_ERR_UNSUPPORTED), (apply(p=-1), cabi.TD_ERR_INVALID_ARG),
    ]
    torch.cuda.synchronize()
    for i, (rc, want) in enumerate(cases):
        assert rc == want, f"case {i}: {rc} ({lib.td_last_error()})"
    torch.cuda.synchronize()
    assert (mean == 7.0).all() and (var == 7.0).all() and (y == 3.0).all()


# ------------------------------------------------------------------------------------------ convolutions
def _post(N, C, seed):
    scale = _rand((N, C), torch.float32, seed) * 0.5 + torch.arange(1, N + 1, device="cuda").view(N, 1).float()
    shift = _rand((N, C), torch.float32, seed + 1) * 3.0 - torch.arange(N, device="cuda").view(N, 1).float() * 10
    return scale.contiguous(), shift.contiguous()


# (H, W) with H * W (or OH * OW) not a multiple of the 128-pixel tile
CONV_CASES = {
    "3x3": dict(k=3, H=13, W=13, cin=128, cout=128),
    "3x3_narrow": dict(k=3, H=21, W=9, cin=256, cout=256),
    "1x1_residual": dict(k=1, H=11, W=19, cin=256, cout=128, res=True),
    "3x3_down": dict(k=3, H=27, W=25, cin=128, cout=128, down=True),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
@pytest.mark.parametrize("dt", list(DTS))
def test_conv_with_per_image_post_constants_is_the_one_image_bits(m, dt, case):
    _, ops, *_ = m
    c = CONV_CASES[case]
    dtype = DTS[dt]
    w = ops.pack_conv_weight(_rand((c["cout"], c["cin"], c["k"], c["k"]), torch.float32, 21) * 0.05, dtype)
    bias = _rand((c["cout"],), torch.float32, 22)
    for N in NS:
        x = _per_image_scaled((N, c["H"], c["W"], c["cin"]), dtype, 100 + N)
        if c.get("down"):
            kw = dict(ksize=3, stride=2, pad=(0, 0), out_hw=((c["H"] - 2) // 2 + 1, (c["W"] - 2) // 2 + 1))
        else:
            kw = dict(ksize=c["k"], pad=(c["k"] // 2, c["k"] // 2))
        oh, ow = kw.get("out_hw", (c["H"], c["W"]))
        assert (oh * ow) % 128 != 0
        res = _rand((N, oh, ow, c["cout"]), dtype, 23) if c.get("res") else None
        scale, shift = _post(N, c["cout"], 30 + N)
        for act in (False, True):
            single = ops.conv2d_nhwc(x, w, bias, residual=res, post=(scale, shift, act), **kw)
            raw, normed = ops.conv2d_nhwc(x, w, bias, residual=res, post=(scale, shift, act), dual=True, **kw)
            for n in range(N):
                r1 = res[n:n + 1] if res is not None else None
                post1 = (scale[n].contiguous(), shift[n].contiguous(), act)
                want = ops.conv2d_nhwc(x[n:n + 1], w, bias, residual=r1, post=post1, **kw)
                want_raw, want_normed = ops.conv2d_nhwc(x[n:n + 1], w, bias, residual=r1, post=post1, dual=True, **kw)
                what = f"{dt} {case} N={N} act={act} image {n}"
                assert_bit_equal(single[n:n + 1], want, what + " single")
                assert_bit_equal(raw[n:n + 1], want_raw, what + " dual raw")
                assert_bit_equal(normed[n:n + 1], want_normed, what + " dual normalised")
        # one shared vector (post_stride 0) is today's form: every image reads row 0
        shared = ops.conv2d_nhwc(x, w, bias, residual=res, post=(scale[0].contiguous(), shift[0].contiguous(), True), **kw)
        broad = ops.conv2d_nhwc(x, w, bias, residual=res, post=(scale[:1].expand(N, -1).contiguous(), shift[:1].expand(N, -1).contiguous(), True), **kw)
        assert_bit_equal(shared, broad, f"{dt} {case} N={N} shared constants")


@pytest.mark.parametrize("dt", list(DTS))
def test_folded_upsample_with_per_image_post_constants_is_the_one_image_bits(m, dt):
    _, ops, *_ = m
    dtype = DTS[dt]
    C = 256
    w16 = ops.fold_upsample_weight(_rand((C, C, 3, 3), torch.float32, 41) * 0.03, dtype)
    bias = _rand((C,), torch.float32, 42)
    for N in NS:
        x = _per_image_scaled((N, 7, 9, C), dtype, 200 + N)          # 14 x 18 output: 252 pixels per image
        scale, shift = _post(N, C, 50 + N)
        for act in (False, True):
            single = ops.upconv2x_nhwc(x, w16, bias, post=(scale, shift, act))
            raw, normed = ops.upconv2x_nhwc(x, w16, bias, post=(scale, shift, act), dual=True)
            for n in range(N):
                post1 = (scale[n].contiguous(), shift[n].contiguous(), act)
                assert_bit_equal(single[n:n + 1], ops.upconv2x_nhwc(x[n:n + 1], w16, bias, post=post1), f"{dt} N={N} image {n}")
                wr, wn = ops.upconv2x_nhwc(x[n:n + 1], w16, bias, post=post1, dual=True)
                assert_bit_equal(raw[n:n + 1], wr, f"{dt} N={N} image {n} dual raw")
                assert_bit_equal(normed[n:n + 1], wn, f"{dt} N={N} image {n} dual normalised")


def test_conv_refuses_bad_post_strides_and_leaves_the_output_untouched(m):
    cabi, ops, *_ = m
    N, H, W, C = 2, 9, 9, 128
    x = _rand((N, H, W, C), torch.float16, 60)
    w = ops.pack_conv_weight(_rand((C, C, 3, 3), torch.float32, 61) * 0.05, torch.float16)
    scale, shift = _post(N, 2 * C, 62)
    y = torch.full((N, H, W, C), 5.0, dtype=torch.float16, device="cuda")

    def call(stride, post=True, per_row=0, up2=False):
        d = cabi.TdConvDesc(N=N, H=H, W=W, Cin=C, Cout=C, kh=3, kw=3, stride=1, pad_top=1, pad_left=1, OH=2 * H if up2 else H,
                            OW=2 * W if up2 else W, dtype=cabi.TD_F16, bias_per_row=per_row, alpha=1.0, x_pitch=C, w_pitch=C, y_pitch=C,
                            res_pitch=0, post_scale=scale.data_ptr() if post else None, post_shift=shift.data_ptr() if post else None,
                            post_act=1, post_stride=stride)
        if up2:
            return cabi.lib.td_upconv2x_nhwc(ctypes.byref(d), x.data_ptr(), w.data_ptr(), None, y.data_ptr(), cabi.current_stream_ptr())
        return cabi.lib.td_conv2d_nhwc(ctypes.byref(d), x.data_ptr(), w.data_ptr(), None, None, y.data_ptr(), cabi.current_stream_ptr())
    for kw in (dict(stride=C - 4), dict(stride=C + 2), dict(stride=-C), dict(stride=C, post=False), dict(stride=C, per_row=1),
               dict(stride=C - 4, up2=True), dict(stride=C + 2, up2=True), dict(stride=C, post=False, up2=True)):
        assert call(**kw) == cabi.TD_ERR_INVALID_ARG, (kw, cabi.lib.td_last_error())
    torch.cuda.synchronize()
    assert (y == 5.0).all()


# ------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("T,C", [(1, 64), (100, 512), (4097, 256), (46341, 512)])
def test_batched_fused_attention_is_the_one_image_bits(m, dt, T, C):
    _, ops, *_ = m
    dtype = DTS[dt]
    for N in (NS if T < 10000 else (2, 3)):
        q, k, v = (_per_image_scaled((N, T, C), dtype, 300 + i + N) for i in range(3))
        got = ops.attention(q, k, v, C ** -0.5)
        for n in range(N):
            assert_bit_equal(got[n], ops.attention(q[n], k[n], v[n], C ** -0.5), f"{dt} T={T} C={C} N={N} image {n}")
        # strided images (a wider row pitch and a gap between images)
        wide = torch.zeros((N, T + 3, C + 64), dtype=dtype, device="cuda")
        wide[:, :T, :C] = q
        out = torch.full((N, T + 1, C + 8), 9.0, dtype=dtype, device="cuda")
        ops.attention(wide[:, :T, :C], k, v, C ** -0.5, out=out[:, :T, :C])
        assert_bit_equal(out[:, :T, :C], got, f"{dt} T={T} C={C} N={N} strided")
        assert (out[:, T:] == 9.0).all() and (out[:, :, C:] == 9.0).all()


def test_batched_attention_refuses_and_leaves_the_output_untouched(m):
    cabi, *_ = m
    N, T, C = 2, 70, 128
    q = _rand((N, T, C), torch.float16, 70)
    o = torch.full((N, T, C), 4.0, dtype=torch.float16, device="cuda")
    s = cabi.current_stream_ptr()

    def call(n=N, t=T, qi=T * C, oi=T * C, qp=q.data_ptr(), op=o.data_ptr(), pitch=C):
        return cabi.lib.td_attention_batched(qp, q.data_ptr(), q.data_ptr(), op, n, t, C, pitch, C, C, C, qi, T * C, T * C, oi, 0.1,
                                             cabi.TD_F16, s)
    for kw in (dict(n=0), dict(n=65536), dict(t=0), dict(qi=T * C - 8), dict(oi=T * C - 8), dict(qi=T * C + 4), dict(oi=-T * C),
               dict(qp=q.data_ptr() + 2), dict(op=o.data_ptr() + 2), dict(op=None), dict(pitch=C + 4)):
        assert call(**kw) == cabi.TD_ERR_INVALID_ARG, (kw, cabi.lib.td_last_error())
    torch.cuda.synchronize()
    assert (o == 4.0).all()


@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("hw", [(13, 11), (216, 216)], ids=["four_gemm", "fused"])
def test_backend_attention_of_a_batch_is_the_one_image_bits(m, dt, hw):
    """TensorCoreBackend.attention on [n, H, W, C]: one projection GEMM over all images, then per image the four-GEMM
    path (below SCORE_MATRIX_MAX_TOKENS) or one fused launch for all images (above it), then proj_out."""
    _, ops, ve, *_ = m
    from oracle import ldm_vae
    dtype = DTS[dt]
    H, W = hw
    assert (H * W > ve.SCORE_MATRIX_MAX_TOKENS) == (hw == (216, 216))
    blk = ldm_vae.seeded_init(ldm_vae.AttnBlock(512), 9).cuda().to(dtype)
    prog = ve.Program([ve.Attention(blk)], 0, True, 1)
    be = ve.TensorCoreBackend(prog, torch.device("cuda"), dtype)
    op = prog.ops[0]
    for N in ((2, 3) if H * W > 10000 else (2, 3, 8)):
        a = _per_image_scaled((N, H, W, 512), dtype, 400 + N)
        skip = _rand((N, H, W, 512), dtype, 401)
        scale, shift = _post(N, 512, 402)
        got = be.attention(a, op, skip)
        raw, normed = be.attention(a, op, skip, post=(scale, shift, True), dual=True)
        for n in range(N):
            s1 = skip[n:n + 1]
            assert_bit_equal(got[n:n + 1], be.attention(a[n:n + 1], op, s1), f"{dt} {hw} N={N} image {n}")
            wr, wn = be.attention(a[n:n + 1], op, s1, post=(scale[n:n + 1], shift[n:n + 1], True), dual=True)
            assert_bit_equal(raw[n:n + 1], wr, f"{dt} {hw} N={N} image {n} dual raw")
            assert_bit_equal(normed[n:n + 1], wn, f"{dt} {hw} N={N} image {n} dual normalised")
        del a, skip, got, raw, normed
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ the hook, end to end
DEC = (40, 52, 8)        # z [N, 4, 40, 52], tile 8: 12 tiles
ENC = (200, 264, 48)     # image [N, 3, 200, 264], tile 48: 15 tiles


def _net(is_dec, dtype):
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), 3 if is_dec else 4)
    net.eval()
    net.original_forward = net.forward
    return net.cuda().to(dtype)


_NETS = {}


def _hook(m, is_dec, dtype, fast=False, color_fix=False):
    tv = m[3]
    key = (is_dec, dtype)
    if key not in _NETS:
        _NETS[key] = _net(is_dec, dtype)
    H, W, tile = DEC if is_dec else ENC
    return tv.VAEHook(_NETS[key], tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=color_fix)


def _input(is_dec, N, dtype, seed):
    from oracle import synth
    H, W, _ = DEC if is_dec else ENC
    x = synth.latent(seed, (N, 4 if is_dec else 3, H, W), torch.float32)
    x[N // 2] *= 100.0          # one image far from the others: a statistic of the wrong image shows
    return x.to("cuda", dtype)


def _decode(hook, x, k, budget=None, wrap=False):
    hook.images_per_pass, hook.max_resident_bytes = k, budget
    hook.wrap_x = hook.wrap_y = wrap
    with torch.no_grad():
        out = hook(x)
    torch.cuda.synchronize()
    return out, dict(hook.last_park_stats)


HOOK_CASES = {
    "dec_slow": dict(is_dec=True),
    "dec_fast": dict(is_dec=True, fast=True),
    "enc_slow": dict(is_dec=False),
    "enc_fast": dict(is_dec=False, fast=True),
    "enc_fast_color_fix": dict(is_dec=False, fast=True, color_fix=True),
    "dec_slow_wrapped": dict(is_dec=True, wrap=True),
    "enc_fast_color_fix_wrapped": dict(is_dec=False, fast=True, color_fix=True, wrap=True),
}


@pytest.mark.parametrize("case", list(HOOK_CASES))
@pytest.mark.parametrize("N", [2, 3, 4])
def test_hook_batched_pass_is_the_one_image_schedule(m, case, N):
    c = dict(HOOK_CASES[case])
    wrap = c.pop("wrap", False)
    dtype = torch.float16 if N != 3 else torch.bfloat16
    hook = _hook(m, dtype=dtype, **c)
    x = _input(c["is_dec"], N, dtype, 17 + N)
    want, st1 = _decode(hook, x, 1, wrap=wrap)
    got, st = _decode(hook, x, None, wrap=wrap)
    assert hook.backend_name == "wgmma"
    assert st1["images_per_pass"] == 1 and st["images_per_pass"] == N, st
    assert_bit_equal(got, want, f"{case} N={N}: chosen k vs k = 1")
    if N == 4:
        mid, _ = _decode(hook, x, 3, wrap=wrap)             # passes of 3 and 1 images
        assert_bit_equal(mid, want, f"{case} N={N}: k = 3")


@pytest.mark.parametrize("is_dec", [True, False], ids=["decoder", "encoder"])
def test_hook_batched_pass_under_parking(m, is_dec):
    """A budget of 0 parks every tile at every barrier: the batched tiles go through pinned host memory and back."""
    hook = _hook(m, is_dec, torch.float16)
    x = _input(is_dec, 3, torch.float16, 5)
    want, _ = _decode(hook, x, 1)
    got, st = _decode(hook, x, 3, budget=0)
    assert st["images_per_pass"] == 3 and sum(st["tiles_parked"].values()) > 0 and st["d2h_bytes"] > 0
    assert_bit_equal(got, want, "parked batched pass vs unbounded k = 1")
    _, st_auto = _decode(hook, x, None, budget=0)
    assert st_auto["images_per_pass"] == 1          # parking under a batched pass is never chosen


def test_hook_nan_in_the_estimate_falls_back_per_image(m, capsys):
    """Fast mode: an image whose estimate meets a NaN runs without frozen statistics.  The batched call then runs its
    group one image at a time, reporting each NaN estimate as the one-image schedule does, and the NaN check of the
    result still refuses it."""
    hook = _hook(m, True, torch.float16, fast=True)
    x = _input(True, 3, torch.float16, 8)
    x[1, :, 3, 5] = float("inf")
    reports = []
    for k in (1, None):
        with pytest.raises(RuntimeError, match="NaN"):
            _decode(hook, x, k)
        reports.append(capsys.readouterr().out.count("Nan detected in fast mode estimation"))
    assert reports[0] > 0 and reports[1] == reports[0], reports


def test_hook_interrupt_in_a_batched_pass_returns_the_partial_result(m):
    tv, host, ve = m[3], m[4], m[2]
    hook = _hook(m, True, torch.float16)
    x = _input(True, 3, torch.float16, 9)
    want, _ = _decode(hook, x, 1)
    real = ve.TensorCoreBackend.paste
    count = [0]

    def paste(self, *a, **kw):
        real(self, *a, **kw)
        count[0] += 1
        if count[0] == 2:
            host.get_shared().state.interrupted = True
    ve.TensorCoreBackend.paste = paste
    try:
        got, st = _decode(hook, x, 3)
    finally:
        ve.TensorCoreBackend.paste = real
        host.get_shared().state.interrupted = False
    assert st["images_per_pass"] == 3
    ib, ob = hook.split_tiles(x.shape[2], x.shape[3])
    for i, b in enumerate(ob):                 # the forward order of the last round: tiles 0 and 1 of all three images
        region = (slice(None), slice(None), slice(b[2], b[3]), slice(b[0], b[1]))
        if i < 2:
            assert_bit_equal(got[region], want[region], f"tile {i}")
        else:
            assert not got[region].any(), f"tile {i} should not have been pasted"


# ------------------------------------------------------------------------------------------ launch counts
_COUNT_JOB = r"""
import json, sys, torch
sys.path.insert(0, "tests")
import test_gpu_vae_batch as t
from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, host, tilevae, vae_engine, vae_ops
m = (_cabi, vae_ops, vae_engine, tilevae, host)
fast = sys.argv[1] == "fast"
hook = t._hook(m, True, torch.float16, fast=fast)
x = t._input(True, 3, torch.float16, 10)
t._decode(hook, x, None)
calls = [0]
real = vae_engine.TensorCoreBackend.attention
def spy(self, a, *args, **kw):
    calls[0] += 1
    return real(self, a, *args, **kw)
vae_engine.TensorCoreBackend.attention = spy
t._decode(hook, x[:1], None)
vae_engine.TensorCoreBackend.attention = real
one = t._conv_launches(lambda: t._decode(hook, x[:1], None))
batched = t._conv_launches(lambda: t._decode(hook, x, None))
k = hook.last_park_stats["images_per_pass"]
per_image = t._conv_launches(lambda: t._decode(hook, x, 1))
print(json.dumps(dict(one=one, batched=batched, per_image=per_image, k=k, attention_calls=calls[0])))
"""


def _conv_launches(fn) -> int:
    """Launches of the convolution kernel in `fn` (CUPTI kernel trace through torch.profiler).  A session counts only when
    both marker kernels around `fn` are in its trace (a session can lose an activity buffer); two complete sessions must
    agree."""
    from torch.profiler import ProfilerActivity, profile
    counts = []
    for _ in range(6):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                kernels = [e.get("name", "") for e in json.load(f).get("traceEvents", []) if e.get("cat") == "kernel"]
        if sum("spin_kernel" in k for k in kernels) < 2:
            continue
        counts.append(sum("conv_gemm_kernel" in k for k in kernels))
        if len(counts) >= 2 and counts[-1] == counts[-2]:
            return counts[-1]
    raise AssertionError(f"no two complete kernel traces agreed: {counts}")


@pytest.mark.parametrize("fast", [False, True], ids=["slow", "fast"])
def test_convolutions_per_pass_do_not_grow_with_the_batch(m, fast):
    """Every convolution (folded upsample included) is one launch for all images of a pass.  The one exception is the
    four-GEMM attention below SCORE_MATRIX_MAX_TOKENS, whose score matrix is per image: its V^T, score and P V GEMMs run
    once per image (3 (N - 1) launches more per attention call).  The traces are taken in a process of their own: a
    profiler session late in a long run can come back without its kernels."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _COUNT_JOB, "fast" if fast else "slow"], cwd=root, capture_output=True, text=True,
                         timeout=900, env=dict(os.environ, PYTHONPATH=root))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    c = json.loads(res.stdout.strip().splitlines()[-1])
    assert c["k"] == 3 and c["attention_calls"] > 0 and c["one"] > 0, c
    assert c["per_image"] == 3 * c["one"], c
    assert c["batched"] == c["one"] + 3 * 2 * c["attention_calls"], c
