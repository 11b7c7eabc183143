"""Tiled-VAE kernels and the VAEHook executor on the GPU against the oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vae
from oracle.make_golden import VAE_CASES, VAE_SUBSAMPLE, vae_case_inputs

pytestmark = pytest.mark.gpu
DT = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}


@pytest.fixture(scope="module")
def tv():
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return tilevae


@pytest.mark.parametrize("shape", [(1, 128, 118, 118), (2, 64, 37, 41), (1, 32, 8, 8), (3, 512, 30, 30), (1, 128, 236, 236)])
@pytest.mark.parametrize("dn", list(DT))
def test_gn_stats_match_torch_var_mean(tv, shape, dn):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(shape, generator=g) * 1.7 + 0.6).to(DT[dn])
    var, mean = tv.get_var_mean(x.cuda(), 32)
    wv, wm = vae.get_var_mean(x.float())
    assert var.dtype == torch.float32 and var.shape == (shape[0] * 32,)
    assert torch.allclose(mean.cpu(), wm, rtol=2e-5, atol=2e-6)
    assert torch.allclose(var.cpu(), wv, rtol=5e-5, atol=1e-6)


def test_gn_stats_large_offset_is_stable(tv):
    """mean^2 >> var: the shifted / Chan-merged moments must not cancel catastrophically."""
    g = torch.Generator().manual_seed(2)
    x = (torch.randn((1, 64, 96, 96), generator=g) * 0.01 + 100.0)
    var, mean = tv.get_var_mean(x.cuda(), 32)
    wv, wm = vae.get_var_mean(x.double())
    assert torch.allclose(var.cpu().double(), wv, rtol=2e-3)
    assert torch.allclose(mean.cpu().double(), wm, rtol=1e-6)


@pytest.mark.parametrize("shape", [(1, 128, 59, 59), (2, 64, 24, 40), (1, 32, 7, 9)])
@pytest.mark.parametrize("dn", list(DT))
@pytest.mark.parametrize("act", [False, True])
def test_gn_apply_matches_reference_formula(tv, shape, dn, act):
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(shape, generator=g) * 2 + 0.3).to(DT[dn])
    C = shape[1]
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    var, mean = vae.get_var_mean(x.float())             # [b*32]; perturbed: "externally supplied" statistics
    var, mean = var * 1.3 + 0.05, mean + 0.1
    want = vae.custom_group_norm(x.float(), mean, var, gamma, beta)
    if act:
        want = F.silu(want)
    got = tv.custom_group_norm(x.cuda(), 32, mean.cuda(), var.cuda(), gamma.cuda(), beta.cuda(), 1e-6, act=act)
    assert got.dtype == DT[dn]
    tol = {"f32": 3e-6, "f16": 2e-3, "bf16": 1.6e-2}[dn]
    assert (got.cpu().float() - want).abs().max() <= tol * max(1.0, want.abs().max().item())


def test_copy_region_crop_and_paste(tv):
    for dt in (torch.float16, torch.float32):
        z = torch.arange(2 * 3 * 40 * 56, dtype=torch.float32).view(2, 3, 40, 56).to(dt).cuda()
        for (y0, y1, x0, x1) in [(0, 16, 0, 24), (5, 33, 7, 50), (8, 40, 8, 56), (39, 40, 55, 56)]:
            t = torch.empty((2, 3, y1 - y0, x1 - x0), dtype=dt, device="cuda")
            tv.copy_region(z[:, :, y0:y1, x0:x1], t)
            assert torch.equal(t, z[:, :, y0:y1, x0:x1])
            canvas = torch.zeros_like(z)
            tv.copy_region(t, canvas[:, :, y0:y1, x0:x1])
            ref = torch.zeros_like(z)
            ref[:, :, y0:y1, x0:x1] = t
            assert torch.equal(canvas, ref)


@pytest.mark.parametrize("H,W,tile", [(128, 128, 96), (40, 52, 16), (97, 333, 64), (1024, 1024, 96)])
def test_nearest_exact_indices_match_torch(tv, H, W, tile):
    scale = tile / max(H, W)
    z = torch.arange(H * W, dtype=torch.float32).view(1, 1, H, W)
    want = F.interpolate(z, scale_factor=scale, mode="nearest-exact")
    oh, sy = tv.nearest_exact_indices(H, scale)
    ow, sx = tv.nearest_exact_indices(W, scale)
    assert (oh, ow) == tuple(want.shape[2:])
    assert torch.equal(z[0, 0][torch.from_numpy(sy).long()][:, torch.from_numpy(sx).long()], want[0, 0])


@pytest.mark.parametrize("dn", ["f32", "f16"])
def test_fast_mode_estimator_input(tv, dn):
    g = torch.Generator().manual_seed(4)
    z = (torch.randn((1, 4, 70, 100), generator=g) * 5 + 1).to(DT[dn])
    want = vae.fast_mode_estimator_input(z.float() if dn == "f32" else z, 32)
    got = tv.fast_mode_estimator_input(z.cuda(), 32)
    assert got.shape == want.shape and got.dtype == z.dtype
    tol = 2e-5 if dn == "f32" else 3e-2
    assert (got.cpu().float() - want.float()).abs().max() <= tol * max(1.0, want.float().abs().max().item())


@pytest.mark.parametrize("case", VAE_CASES, ids=[c[0] for c in VAE_CASES])
def test_vaehook_fp32_matches_oracle_and_reference_fixture(tv, golden_dir, case):
    import os
    name, is_dec, fast, cf, H, W, tile = case
    net, z = vae_case_inputs(is_dec, H, W)
    with torch.no_grad():
        want = vae.vae_hook_call(net, z, tile, is_dec, fast, cf)
    net_gpu, _ = vae_case_inputs(is_dec, H, W)
    net_gpu = net_gpu.cuda()
    net_gpu.original_forward = net_gpu.forward
    hook = tv.VAEHook(net_gpu, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=cf)
    with torch.no_grad():
        got = hook(z.cuda())
    assert got.shape == want.shape and got.dtype == torch.float32
    scale = max(1.0, want.abs().max().item())
    err = (got.cpu() - want).abs().max().item()
    assert err <= 3e-4 * scale, f"{name}: max err {err} vs scale {scale}"
    g = np.load(os.path.join(golden_dir, "vae_small.npz"))
    sub = got.cpu()[:, :, ::VAE_SUBSAMPLE, ::VAE_SUBSAMPLE].numpy()
    assert np.abs(sub - g[name]).max() <= 3e-4 * scale, f"{name}: differs from the reference's own output"
    if H > 2 * hook.pad + tile:
        assert tuple(net_gpu.last_z_shape) == tuple(z.shape)


@pytest.mark.parametrize("is_dec,fast", [(True, True), (True, False), (False, True)])
def test_vaehook_fp16_close_to_fp32_oracle(tv, is_dec, fast):
    H, W, tile = (40, 52, 16) if is_dec else (200, 264, 64)
    net, z = vae_case_inputs(is_dec, H, W)
    with torch.no_grad():
        want = vae.vae_hook_call(net, z, tile, is_dec, fast, False)
    net16, _ = vae_case_inputs(is_dec, H, W)
    net16 = net16.cuda().half()
    hook = tv.VAEHook(net16, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
    with torch.no_grad():
        got = hook(z.cuda().half())
    assert got.dtype == torch.float16
    diff = (got.cpu().float() - want).abs()
    scale = want.abs().max().item()
    assert diff.mean().item() <= 4e-3 * scale and diff.max().item() <= 6e-2 * scale


def test_vaehook_batch_of_two(tv):
    net, z = vae_case_inputs(True, 40, 52)
    z2 = torch.cat([z, z.flip(3)], dim=0)
    with torch.no_grad():
        want = vae.vae_hook_call(net, z2, 16, True, False, False)
    net_gpu, _ = vae_case_inputs(True, 40, 52)
    hook = tv.VAEHook(net_gpu.cuda(), 16, True, False, False, False)
    with torch.no_grad():
        got = hook(z2.cuda())
    assert (got.cpu() - want).abs().max().item() <= 3e-4 * max(1.0, want.abs().max().item())


# ------------------------------------------------------------------------------- tensor-core backend (fp16 / bf16 networks)
def _sd_width_net(is_dec, seed):
    """Full-width SD autoencoder half (ch=128, ch_mult (1,2,4,4), 2 res blocks): the layer shapes of BASELINE cfg4."""
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), seed)
    net.eval()
    net.original_forward = net.forward
    return net


@pytest.mark.parametrize("is_dec,fast,H,W,tile", [(True, True, 40, 52, 16), (True, False, 40, 52, 16), (False, True, 200, 264, 64), (False, False, 136, 200, 64)])
def test_vaehook_tensor_core_backend_matches_fp32_reference(tv, is_dec, fast, H, W, tile):
    """fp16 network on the wgmma / channels-last backend vs the fp32 restatement of the reference's tiled algorithm
    (oracle, run on the GPU in fp32: same tiles, same statistics merge).  fp16 activations through ~60 layers:
    mean error <= 2e-3 * scale, max <= 3e-2 * scale."""
    from oracle import synth
    net = _sd_width_net(is_dec, 3 if is_dec else 4)
    z = synth.latent(5 if is_dec else 6, (1, 4 if is_dec else 3, H, W), torch.float32)
    ref_net = _sd_width_net(is_dec, 3 if is_dec else 4).cuda()
    with torch.no_grad():
        want = vae.vae_hook_call(ref_net, z.cuda(), tile, is_dec, fast, False).cpu()
    net16 = net.cuda().half()
    hook = tv.VAEHook(net16, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
    with torch.no_grad():
        got = hook(z.cuda().half())
    assert hook.backend_name == "wgmma"
    assert got.dtype == torch.float16 and got.shape == want.shape
    diff = (got.cpu().float() - want).abs()
    scale = want.abs().max().item()
    assert diff.mean().item() <= 2e-3 * scale and diff.max().item() <= 3e-2 * scale, (diff.mean().item() / scale, diff.max().item() / scale)


def test_tensor_core_backend_matches_module_backend_on_the_same_fp16_network(tv):
    """Same fp16 weights, same tiles: wgmma / channels-last backend vs cuDNN modules + NCHW kernels."""
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    from oracle import synth
    net16 = _sd_width_net(True, 3).cuda().half()
    z = synth.latent(5, (1, 4, 40, 52), torch.float16).cuda()
    hook = tv.VAEHook(net16, 16, True, True, True, False)
    with torch.no_grad():
        a = hook(z)
        orig = ve.pick_backend
        ve.pick_backend = lambda program, device, dtype: ve.ModuleBackend(program, device, dtype)
        try:
            b = hook(z)
        finally:
            ve.pick_backend = orig
    assert hook.backend_name == "modules"
    scale = b.float().abs().max().item()
    d = (a.float() - b.float()).abs()
    assert d.mean().item() <= 1e-3 * scale and d.max().item() <= 2e-2 * scale
