"""Parity of the wgmma implicit-GEMM convolution / GEMM (csrc/td_conv.cu) and the channels-last streaming kernels
(csrc/td_nhwc.cu) against plain PyTorch fp32 references of the same ops.  Tolerances: fp16 / bf16 inputs, fp32
accumulation, output rounded once to the activation dtype -> |err| <= 1e-3 * scale for fp16 (SURVEY / VERDICT bar),
8e-3 * scale for bf16 (8 mantissa bits)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 1e-3, torch.bfloat16: 8e-3}


@pytest.fixture(scope="module")
def ops():
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops
    return vae_ops


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * scale).to(dtype)


def _check(got, want, dtype, what):
    scale = want.abs().max().item() + 1e-6
    err = (got.float() - want).abs().max().item()
    assert err <= TOL[dtype] * scale, f"{what}: max err {err:.4g} vs scale {scale:.4g} (rel {err / scale:.3g})"


@pytest.mark.parametrize("M,K,N", [(128, 64, 128), (256, 128, 256), (384, 512, 64), (1000, 192, 520), (130, 64, 16)])
def test_gemm_nt(ops, M, K, N):
    dtype = torch.float16
    a, b = _rand((M, K), dtype, 1, 0.5), _rand((N, K), dtype, 2, 0.5)
    got = ops.gemm_nt(a, b)
    _check(got, a.float() @ b.float().t(), dtype, f"gemm {M}x{K}x{N}")


def test_gemm_alpha_bias_rows_and_padded_pitch(ops):
    dtype = torch.float16
    M, K, N = 300, 200, 264          # K not a multiple of 64: the operands sit in zero-padded wider buffers
    Kp = 256
    a = torch.zeros((M, Kp), dtype=dtype, device="cuda"); a[:, :K] = _rand((M, K), dtype, 3, 0.5)
    b = torch.zeros((N, Kp), dtype=dtype, device="cuda"); b[:, :K] = _rand((N, K), dtype, 4, 0.5)
    bias = _rand((M,), torch.float32, 5)
    got = ops.gemm_nt(a, b, bias=bias, alpha=0.125, bias_per_row=True)
    want = 0.125 * (a.float() @ b.float().t()) + bias[:, None]
    _check(got, want, dtype, "gemm alpha/bias-per-row")
    bias_c = _rand((N,), torch.float32, 6)
    got = ops.gemm_nt(a, b, bias=bias_c)
    _check(got, a.float() @ b.float().t() + bias_c[None, :], dtype, "gemm bias-per-col")


def _conv_case(ops, dtype, N, H, W, Cin, Cout, k, stride, seed, residual=False, cin_real=None):
    cin_real = cin_real or Cin
    x = _rand((N, cin_real, H, W), dtype, seed, 0.7)
    w = _rand((Cout, cin_real, k, k), dtype, seed + 1, 1.0 / (cin_real * k * k) ** 0.5)
    bias = _rand((Cout,), torch.float32, seed + 2, 0.3)
    if stride == 1:
        want = F.conv2d(x.float(), w.float(), bias, stride=1, padding=k // 2)
        pad, out_hw = (k // 2, k // 2), (H, W)
    else:   # ldm Downsample: pad (0,1,0,1) then 3x3 stride 2, no conv padding
        want = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), w.float(), bias, stride=2, padding=0)
        pad, out_hw = (0, 0), (want.shape[2], want.shape[3])
    xn = ops.nchw_to_nhwc(x, Cin)
    wp = ops.pack_conv_weight(w, dtype, cin_pad=Cin)
    res = None
    if residual:
        res = _rand((N, out_hw[0], out_hw[1], Cout), dtype, seed + 3, 0.5)
        want = want + res.float().permute(0, 3, 1, 2)
    got = ops.conv2d_nhwc(xn, wp, bias, ksize=k, stride=stride, pad=pad, out_hw=out_hw, residual=res)
    _check(got.permute(0, 3, 1, 2), want, dtype, f"conv {(N, H, W, Cin, Cout, k, stride)} {dtype}")


def test_conv1x1(ops):
    _conv_case(ops, torch.float16, 1, 24, 40, 64, 128, 1, 1, 10)


def test_conv3x3_small(ops):
    _conv_case(ops, torch.float16, 1, 16, 16, 64, 64, 3, 1, 20)


def test_conv3x3_odd_sizes_and_residual(ops):
    _conv_case(ops, torch.float16, 1, 33, 75, 128, 128, 3, 1, 30, residual=True)


def test_conv3x3_two_cout_blocks(ops):
    _conv_case(ops, torch.float16, 1, 40, 52, 128, 512, 3, 1, 40)


def test_conv3x3_batch_and_bf16(ops):
    _conv_case(ops, torch.bfloat16, 2, 20, 36, 64, 256, 3, 1, 50, residual=True)


def test_conv_padded_input_channels(ops):
    # conv_in: 4 real channels zero-padded to 64
    _conv_case(ops, torch.float16, 1, 30, 30, 64, 128, 3, 1, 60, cin_real=4)


def test_conv_narrow_output(ops):
    # conv_out: 3 output channels (padded to 16 rows of weights / 16-wide MMA)
    dtype = torch.float16
    x = _rand((1, 128, 28, 44), dtype, 70, 0.7)
    w = _rand((3, 128, 3, 3), dtype, 71, 0.03)
    bias = _rand((3,), torch.float32, 72, 0.3)
    want = F.conv2d(x.float(), w.float(), bias, padding=1)
    xn = ops.nchw_to_nhwc(x, 128)
    wp = ops.pack_conv_weight(w, dtype, cout_pad=16)
    b16 = torch.zeros(16, dtype=torch.float32, device="cuda"); b16[:3] = bias
    got = ops.conv2d_nhwc(xn, wp, b16, ksize=3, pad=(1, 1), cout=16)
    _check(got[..., :3].permute(0, 3, 1, 2), want, dtype, "conv_out")
    assert float(got[..., 3:].abs().max()) == 0.0


def test_conv3x3_stride2_downsample(ops):
    _conv_case(ops, torch.float16, 1, 32, 48, 128, 128, 3, 2, 80)
    _conv_case(ops, torch.float16, 1, 31, 45, 64, 64, 3, 2, 90)


def test_layout_kernels(ops):
    dtype = torch.float16
    x = _rand((2, 5, 19, 23), dtype, 100)
    big = torch.zeros((2, 5, 30, 40), dtype=dtype, device="cuda")
    big[:, :, 4:23, 7:30] = x
    y = ops.nchw_to_nhwc(big[:, :, 4:23, 7:30], 8)
    assert torch.equal(y[..., :5], x.permute(0, 2, 3, 1)) and float(y[..., 5:].abs().max()) == 0.0
    dst = torch.zeros((2, 3, 50, 60), dtype=dtype, device="cuda")
    ops.nhwc_to_nchw_region(y[:, 2:12, 3:20, :], dst[:, :, 5:15, 6:23], 3)
    assert torch.equal(dst[:, :, 5:15, 6:23], x[:, :3, 2:12, 3:20])
    assert float(dst[:, :, :5].abs().max()) == 0.0
    u = ops.upsample2x_nhwc(y)
    assert torch.equal(u.permute(0, 3, 1, 2), F.interpolate(y.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest").to(dtype))


@pytest.mark.parametrize("C", [128, 256, 512])
def test_group_norm_nhwc(ops, C):
    dtype = torch.float16
    x = (_rand((1, C, 37, 53), dtype, 110 + C, 1.3).float() + 0.8).to(dtype)
    xn = x.permute(0, 2, 3, 1).contiguous()
    var, mean = ops.gn_stats_nhwc(xn)
    wv, wm = torch.var_mean(x.float().view(1, 32, -1), dim=2, unbiased=False)
    assert (mean - wm[0]).abs().max() <= 5e-5 * (wm.abs().max() + 1)
    assert ((var - wv[0]).abs() / wv[0]).max() <= 5e-5
    gamma, beta = _rand((C,), torch.float32, 5, 0.5) + 1.0, _rand((C,), torch.float32, 6, 0.2)
    for act in (False, True):
        got = ops.gn_apply_nhwc(xn, mean, var, gamma, beta, act)
        want = F.group_norm(x.float(), 32, gamma, beta, eps=1e-6)
        if act:
            want = F.silu(want)
        _check(got.permute(0, 3, 1, 2), want, dtype, f"gn apply C={C} act={act}")


def test_softmax_rows(ops):
    dtype = torch.float16
    rows, cols, pitch = 37, 1003, 1008
    x = torch.full((rows, pitch), 77.0, dtype=dtype, device="cuda")       # garbage in the padding columns
    x[:, :cols] = _rand((rows, cols), dtype, 120, 3.0)
    y = ops.softmax_rows(x, cols)
    want = torch.softmax(x[:, :cols].float(), dim=1)
    assert (y[:, :cols].float() - want).abs().max() <= 1e-3 * want.max()
    assert float(y[:, cols:].abs().max()) == 0.0


def test_conv3x3_large_grid(ops):
    """Enough pixel tiles (>= 4 per SM) that every persistent CTA walks many (pixel tile, Cout block) pairs through the
    shared-memory ring; odd sizes leave partial tiles."""
    _conv_case(ops, torch.float16, 1, 259, 333, 128, 256, 3, 1, 200, residual=True)   # 21 x 33 = 693 sub-tiles, BN 256
    _conv_case(ops, torch.float16, 1, 253, 336, 64, 128, 3, 1, 210)                   # BN 128
    _conv_case(ops, torch.float16, 1, 663, 541, 64, 64, 3, 2, 220)                    # stride 2 with the doubled box (714 output sub-tiles)
    _conv_case(ops, torch.float16, 1, 200, 248, 64, 512, 3, 1, 230)                   # two Cout blocks of 256
    _conv_case(ops, torch.float16, 1, 330, 270, 128, 256, 3, 2, 240)                  # stride 2, BN 256, small grid
    _conv_case(ops, torch.float16, 1, 660, 540, 64, 256, 3, 2, 250)                   # stride 2, BN 256, 714 sub-tiles
    _conv_case(ops, torch.float16, 1, 397, 403, 64, 128, 3, 1, 260, residual=True)    # BN 128, 1300 tiles


def test_gemm_large_m(ops):
    dtype = torch.float16
    for M in (80003, 160001):       # 626 / 1251 row tiles of 128: several per CTA, a partial last one
        K, N = 64, 128
        a, b = _rand((M, K), dtype, 1, 0.5), _rand((N, K), dtype, 2, 0.5)
        bias = _rand((M,), torch.float32, 5)
        got = ops.gemm_nt(a, b, bias=bias, bias_per_row=True)
        _check(got, a.float() @ b.float().t() + bias[:, None], dtype, f"gemm M={M}")


@pytest.mark.parametrize("act", [False, True])
def test_conv_with_fused_frozen_group_norm(ops, act):
    """conv -> GroupNorm(statistics given) (+ SiLU) in the conv's epilogue == the two ops in fp32."""
    dtype = torch.float16
    N, H, W, Cin, Cout = 1, 37, 45, 128, 256
    x = _rand((N, Cin, H, W), dtype, 300, 0.7)
    w = _rand((Cout, Cin, 3, 3), dtype, 301, 1.0 / (Cin * 9) ** 0.5)
    bias = _rand((Cout,), torch.float32, 302, 0.3)
    res = _rand((N, H, W, Cout), dtype, 303, 0.5)
    gamma, beta = _rand((Cout,), torch.float32, 304, 0.4) + 1.0, _rand((Cout,), torch.float32, 305, 0.2)
    mean, var = _rand((32,), torch.float32, 306, 0.3), _rand((32,), torch.float32, 307, 0.2).abs() + 0.5
    y = F.conv2d(x.float(), w.float(), bias, padding=1) + res.float().permute(0, 3, 1, 2)
    cpg = Cout // 32
    want = (y - mean.repeat_interleave(cpg).view(1, -1, 1, 1)) / torch.sqrt(var.repeat_interleave(cpg).view(1, -1, 1, 1) + 1e-6)
    want = want * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)
    if act:
        want = F.silu(want)
    rstd = (1.0 / torch.sqrt(var + 1e-6)).repeat_interleave(cpg)
    scale = (rstd * gamma).contiguous()
    shift = (beta - mean.repeat_interleave(cpg) * scale).contiguous()
    got = ops.conv2d_nhwc(ops.nchw_to_nhwc(x, Cin), ops.pack_conv_weight(w, dtype), bias, ksize=3, pad=(1, 1), residual=res, post=(scale, shift, act))
    _check(got.permute(0, 3, 1, 2), want, dtype, f"conv + frozen GroupNorm act={act}")


def _upconv_case(ops, dtype, N, H, W, Cin, Cout, seed):
    x = _rand((N, Cin, H, W), dtype, seed, 0.7)
    w = _rand((Cout, Cin, 3, 3), dtype, seed + 1, 1.0 / (Cin * 9) ** 0.5)
    bias = _rand((Cout,), torch.float32, seed + 2, 0.3)
    want = F.conv2d(F.interpolate(x.float(), scale_factor=2.0, mode="nearest"), w.float(), bias, padding=1)
    got = ops.upconv2x_nhwc(ops.nchw_to_nhwc(x, Cin), ops.fold_upsample_weight(w, dtype), bias)
    assert got.shape == (N, 2 * H, 2 * W, Cout)
    # the folded taps are rounded to the activation dtype after the fp32 sum: one more rounding of the weights than the
    # reference's own fp16 weights carry -- same order as the input rounding, inside the same bar
    _check(got.permute(0, 3, 1, 2), want, dtype, f"upsample2x+conv {N}x{Cin}x{H}x{W}->{Cout}")
    # and against the unfolded path on the same kernels (upsample kernel + 3x3 conv)
    ref = ops.conv2d_nhwc(ops.upsample2x_nhwc(ops.nchw_to_nhwc(x, Cin)), ops.pack_conv_weight(w, dtype), bias, ksize=3, pad=(1, 1))
    _check(got, ref.float(), dtype, "folded vs materialised upsample")


@pytest.mark.parametrize("shape", [(1, 8, 8, 64, 64), (1, 37, 45, 128, 128), (2, 19, 23, 256, 256), (1, 64, 9, 64, 512)])
def test_upsample_folded_into_conv(ops, shape):
    N, H, W, Cin, Cout = shape
    _upconv_case(ops, torch.float16, N, H, W, Cin, Cout, 400 + H)


def test_upsample_folded_into_conv_large_pair_and_bf16(ops):
    _upconv_case(ops, torch.float16, 1, 236, 236, 512, 512, 431)     # the decoder's 236 -> 472 block: CTA pairs
    _upconv_case(ops, torch.bfloat16, 1, 120, 130, 128, 128, 437)    # two sub-tiles per CTA


def test_upsample_folded_with_fused_group_norm(ops):
    dtype = torch.float16
    N, H, W, Cin, Cout = 1, 21, 30, 128, 128
    x = _rand((N, Cin, H, W), dtype, 450, 0.7)
    w = _rand((Cout, Cin, 3, 3), dtype, 451, 1.0 / (Cin * 9) ** 0.5)
    bias = _rand((Cout,), torch.float32, 452, 0.3)
    scale, shift = _rand((Cout,), torch.float32, 453, 0.4) + 1.0, _rand((Cout,), torch.float32, 454, 0.2)
    y = F.conv2d(F.interpolate(x.float(), scale_factor=2.0, mode="nearest"), w.float(), bias, padding=1)
    want = F.silu(y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    got = ops.upconv2x_nhwc(ops.nchw_to_nhwc(x, Cin), ops.fold_upsample_weight(w, dtype), bias, post=(scale, shift, True))
    _check(got.permute(0, 3, 1, 2), want, dtype, "upsample2x+conv + affine + SiLU")


@pytest.mark.parametrize("shape", [(1, 37, 45, 128, 128, False), (1, 130, 140, 128, 256, True), (2, 16, 24, 256, 64, True)])
def test_conv_two_outputs_raw_and_normalised(ops, shape):
    """One launch, two tensors: the result before the frozen-GroupNorm stage (next block's shortcut source) and after it."""
    dtype = torch.float16
    N, H, W, Cin, Cout, with_res = shape
    x = _rand((N, Cin, H, W), dtype, 500, 0.7)
    w = _rand((Cout, Cin, 3, 3), dtype, 501, 1.0 / (Cin * 9) ** 0.5)
    bias = _rand((Cout,), torch.float32, 502, 0.3)
    res = _rand((N, H, W, Cout), dtype, 503, 0.5) if with_res else None
    scale, shift = _rand((Cout,), torch.float32, 504, 0.4) + 1.0, _rand((Cout,), torch.float32, 505, 0.2)
    y = F.conv2d(x.float(), w.float(), bias, padding=1)
    if with_res:
        y = y + res.float().permute(0, 3, 1, 2)
    z = F.silu(y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    raw, normed = ops.conv2d_nhwc(ops.nchw_to_nhwc(x, Cin), ops.pack_conv_weight(w, dtype), bias, ksize=3, pad=(1, 1), residual=res,
                                  post=(scale, shift, True), dual=True)
    _check(raw.permute(0, 3, 1, 2), y, dtype, "raw output")
    _check(normed.permute(0, 3, 1, 2), z, dtype, "normalised output")
    # and the single-output forms give the same bits
    only_raw = ops.conv2d_nhwc(ops.nchw_to_nhwc(x, Cin), ops.pack_conv_weight(w, dtype), bias, ksize=3, pad=(1, 1), residual=res)
    only_post = ops.conv2d_nhwc(ops.nchw_to_nhwc(x, Cin), ops.pack_conv_weight(w, dtype), bias, ksize=3, pad=(1, 1), residual=res,
                                post=(scale, shift, True))
    assert torch.equal(raw, only_raw) and torch.equal(normed, only_post)


def test_upsample_folded_two_outputs(ops):
    dtype = torch.float16
    N, H, W, Cin, Cout = 1, 59, 61, 256, 256
    x = _rand((N, Cin, H, W), dtype, 520, 0.7)
    w = _rand((Cout, Cin, 3, 3), dtype, 521, 1.0 / (Cin * 9) ** 0.5)
    bias = _rand((Cout,), torch.float32, 522, 0.3)
    scale, shift = _rand((Cout,), torch.float32, 523, 0.4) + 1.0, _rand((Cout,), torch.float32, 524, 0.2)
    y = F.conv2d(F.interpolate(x.float(), scale_factor=2.0, mode="nearest"), w.float(), bias, padding=1)
    z = F.silu(y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    raw, normed = ops.upconv2x_nhwc(ops.nchw_to_nhwc(x, Cin), ops.fold_upsample_weight(w, dtype), bias, post=(scale, shift, True), dual=True)
    _check(raw.permute(0, 3, 1, 2), y, dtype, "raw output")
    _check(normed.permute(0, 3, 1, 2), z, dtype, "normalised output")
