"""Fused attention (vae_ops.attention, csrc/td_attn.cu) against fp32 torch and the four-GEMM path, its memory bound, and
the tensor-core VAE backend's choice between the two at the reference's large tile sizes."""
import pytest
import torch

pytestmark = pytest.mark.gpu
C = 512
TOL = {torch.float16: 1e-3, torch.bfloat16: 8e-3}      # the GEMM bars of test_gpu_conv.py, relative to max |reference|


@pytest.fixture(scope="module")
def ops():
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_ops
    torch.backends.cuda.matmul.allow_tf32 = False
    return vae_ops


def _qkv(T, dtype, seed):
    """q, k with entries of std 1.7: logits alpha q.k of std ~2.9, a softmax far from uniform."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn((T, C), generator=g, device="cuda") * 1.7).to(dtype)
    k = (torch.randn((T, C), generator=g, device="cuda") * 1.7 + 0.2).to(dtype)
    v = torch.randn((T, C), generator=g, device="cuda").to(dtype)
    return q, k, v


def _reference(q, k, v, alpha, rows=2048):
    """fp32 softmax(alpha q k^T) v, 2048 query rows at a time (never a full T x T matrix)."""
    k32, v32 = k.float(), v.float()
    out = torch.empty(q.shape, dtype=torch.float32, device=q.device)
    for r0 in range(0, q.shape[0], rows):
        s = (q[r0:r0 + rows].float() @ k32.T) * alpha
        out[r0:r0 + rows] = torch.softmax(s, dim=1) @ v32
        del s
    return out


@pytest.mark.parametrize("T", [1517, 4761, 13924, 77284])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_attention_matches_fp32_torch(ops, T, dtype):
    q, k, v = _qkv(T, dtype, 11)
    alpha = C ** -0.5
    got = ops.attention(q, k, v, alpha)
    want = _reference(q, k, v, alpha)
    assert got.dtype == dtype and got.shape == (T, C)
    scale = want.abs().max().item()
    err = (got.float() - want).abs().max().item()
    assert err <= TOL[dtype] * scale, (err / scale, T)


def test_attention_pitched_views(ops):
    """Row pitches wider than C (views into wider buffers) and a T that is not a multiple of 64."""
    T = 1000
    q, k, v = _qkv(T, torch.float16, 12)
    wide = torch.zeros((3, T, C + 64), dtype=torch.float16, device="cuda")
    wide[0, :, :C], wide[1, :, :C], wide[2, :, :C] = q, k, v
    out = torch.zeros((T, C + 128), dtype=torch.float16, device="cuda")
    ops.attention(wide[0, :, :C], wide[1, :, :C], wide[2, :, :C], 0.05, out=out[:, :C])
    want = _reference(q, k, v, 0.05)
    assert (out[:, :C].float() - want).abs().max().item() <= 1e-3 * want.abs().max().item()
    assert torch.count_nonzero(out[:, C:]) == 0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_attention_matches_four_gemm_path(ops, dtype):
    """The same q / k / v through the path TensorCoreBackend keeps for small tiles: S = alpha Q K^T, row softmax, P V.
    That path rounds S to the storage dtype before the softmax, so it is the less accurate of the two: the fused result
    is held to the fp32 bar and to no more error than the four-GEMM result."""
    T = 13924
    q, k, v = _qkv(T, dtype, 13)
    alpha = C ** -0.5
    Tp = ops.round_up(T, 8)
    vt = torch.zeros((C, Tp), dtype=dtype, device="cuda")
    vt[:, :T] = v.T
    s = torch.empty((T, Tp), dtype=dtype, device="cuda")
    ops.gemm_nt(q, k, alpha=alpha, out=s[:, :T])
    ops.softmax_rows(s, T, out=s)
    old = ops.gemm_nt(s, vt)
    del s
    new = ops.attention(q, k, v, alpha)
    want = _reference(q, k, v, alpha)
    scale = want.abs().max().item()
    err_new = (new.float() - want).abs().max().item()
    err_old = (old.float() - want).abs().max().item()
    assert err_new <= TOL[dtype] * scale and err_new <= err_old, (err_new / scale, err_old / scale)


def test_attention_memory_stays_within_its_operands(ops):
    """At the reference's H100 decoder tile (256: 77 284 tokens) the four-GEMM path would need an 11 GiB score matrix;
    the fused call allocates its output and nothing else of note."""
    T = 77284
    q, k, v = _qkv(T, torch.float16, 14)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = ops.attention(q, k, v, C ** -0.5)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    assert rise <= 2 * T * C * 2, rise
    assert torch.isfinite(out).all()


def test_attention_rejects_unsupported_channels(ops):
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_ERR_UNSUPPORTED, TdError
    q = torch.zeros((100, 576), dtype=torch.float16, device="cuda")
    with pytest.raises(TdError) as e:
        ops.attention(q, q, q, 1.0)
    assert e.value.status == TD_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------- VAEHook at the reference's tile sizes
def _sd_width_net(is_dec, seed):
    """Full-width SD autoencoder half (ch=128, ch_mult (1,2,4,4), 2 res blocks), as in test_gpu_vae.py."""
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), seed)
    net.eval()
    net.original_forward = net.forward
    return net


@pytest.fixture
def fused_calls(monkeypatch):
    """Token counts of every fused attention call the tensor-core backend makes."""
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    calls = []
    real = ve.ops.attention

    def spy(q, *a, **kw):
        calls.append(q.shape[0])
        return real(q, *a, **kw)
    monkeypatch.setattr(ve.ops, "attention", spy)
    return calls


def test_tile_below_the_bound_keeps_the_four_gemm_path(fused_calls, monkeypatch):
    """Decoder tile 256 on a 400 x 400 latent: the largest tile has 45 796 tokens, under the bound, and runs the four-GEMM
    path.  Only fast mode's estimator pass (one 256 x 256 tile = 65 536 tokens) is above it."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    from oracle import synth
    four_gemm = []
    real = ve.ops.softmax_rows

    def spy(x, cols, *a, **kw):
        four_gemm.append(cols)
        return real(x, cols, *a, **kw)
    monkeypatch.setattr(ve.ops, "softmax_rows", spy)
    net16 = _sd_width_net(True, 3).cuda().half()
    z = synth.latent(5, (1, 4, 400, 400), torch.float16).cuda()
    hook = tilevae.VAEHook(net16, 256, True, True, True, False)
    with torch.no_grad():
        out = hook(z)
    assert hook.backend_name == "wgmma" and out.shape == (1, 3, 3200, 3200)
    assert max(four_gemm) == 45796 and all(t <= ve.SCORE_MATRIX_MAX_TOKENS for t in four_gemm)
    assert fused_calls == [256 * 256]


def _compare_with_module_backend(hook, x):
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    with torch.no_grad():
        a = hook(x)
        assert hook.backend_name == "wgmma"
        orig = ve.pick_backend
        ve.pick_backend = lambda program, device, dtype: ve.ModuleBackend(program, device, dtype)
        try:
            b = hook(x)
        finally:
            ve.pick_backend = orig
    assert hook.backend_name == "modules"
    scale = b.float().abs().max().item()
    d = (a.float() - b.float()).abs()
    assert d.mean().item() <= 1e-3 * scale and d.max().item() <= 2e-2 * scale, (d.mean().item() / scale, d.max().item() / scale)


def test_decoder_tile_256_takes_the_fused_path_and_matches_module_backend(fused_calls):
    """[1, 4, 520, 260] at the reference's H100 decoder tile (256): the mid-block tiles have up to 72 280 tokens."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from oracle import synth
    net16 = _sd_width_net(True, 3).cuda().half()
    z = synth.latent(5, (1, 4, 520, 260), torch.float16).cuda()
    hook = tilevae.VAEHook(net16, 256, True, True, True, False)
    _compare_with_module_backend(hook, z)
    assert fused_calls and max(fused_calls) == 72280


def test_encoder_tile_2048_takes_the_fused_path_and_matches_module_backend(fused_calls):
    """[1, 3, 2048, 4096] image at encoder tile 2048: the mid-block tiles have up to 66 560 tokens."""
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    from oracle import synth
    net16 = _sd_width_net(False, 4).cuda().half()
    x = synth.latent(6, (1, 3, 2048, 4096), torch.float16).cuda()
    hook = tilevae.VAEHook(net16, 2048, False, True, True, False)
    _compare_with_module_backend(hook, x)
    assert fused_calls and max(fused_calls) == 66560
