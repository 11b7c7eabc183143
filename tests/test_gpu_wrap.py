"""Seamless tiling on the GPU: the wrap scatter / blend kernels (csrc/td_wrap.cu) bit for bit against tests/wrap_oracle.py, the
MultiDiffusion and Mixture of Diffusers delegates on wrapped grids, and the seam property itself."""
import types

import numpy as np
import pytest
import torch

import wrap_oracle as wo
from helpers import DTYPES, assert_bit_equal, region_composite_reference

pytestmark = pytest.mark.gpu

# (w, h, tile_w, tile_h, overlap, tile_bs): W a multiple of every vector width / not (generic kernels)
# (120, 64, 40, 24, 8): periodic origins 0, 30, 60, 90 -- unaligned vector windows, some crossing the seam, in every dtype
SHAPES = [(64, 48, 16, 16, 8, 4), (128, 96, 48, 40, 16, 5), (100, 37, 33, 20, 8, 3), (120, 64, 40, 24, 8, 4)]
WRAPS = [wo.WRAP_X, wo.WRAP_Y, wo.WRAP_X | wo.WRAP_Y]


def _setup(shape, wrap, dn, gaussian=False, N=2, C=4, seed=0):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    w, h, tw, th, ov, bs = shape
    g = engine.make_grid(w, h, tw, th, ov, bs, wrap=wrap)
    plan = wo.WrapPlan(w, h, tw, th, ov, bs, wrap, gaussian)
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn((N, C, h, w), generator=gen) * 2).to(DTYPES[dn])
    return g, plan, x


def _tile_outs(plan, x, seed):
    gen = torch.Generator().manual_seed(seed)
    N, C = x.shape[:2]
    return [(torch.randn((len(bbs) * N, C, plan.tile_h, plan.tile_w), generator=gen) * 1.5).to(x.dtype) for bbs in plan.batched_bboxes]


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wrap", WRAPS)
@pytest.mark.parametrize("shape", SHAPES)
def test_scatter_bit_exact(dn, wrap, shape):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_FLAG_FORCE_GENERIC
    g, plan, x = _setup(shape, wrap, dn)
    want = wo.scatter(x, plan.bboxes)
    xd = x.cuda()
    assert_bit_equal(engine.scatter_tiles(g, xd).cpu(), want, f"wrap scatter {dn} {wrap} {shape}")
    assert_bit_equal(engine.scatter_tiles(g, xd, flags=TD_FLAG_FORCE_GENERIC).cpu(), want, "generic")
    T, N = g.num_tiles, x.shape[0]
    b, e = T // 3, T - 1                                  # a tile sub-range (the tile shard's / icond crop's form)
    assert_bit_equal(engine.scatter_tiles(g, xd, tile_begin=b, tile_end=e).cpu(), want[b * N:e * N], "sub-range")


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wrap", WRAPS)
@pytest.mark.parametrize("shape", SHAPES)
def test_blend_multidiffusion_bit_exact(dn, wrap, shape):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_FLAG_FORCE_GENERIC
    g, plan, x = _setup(shape, wrap, dn, seed=1)
    N, C = x.shape[:2]
    outs = _tile_outs(plan, x, 2)
    want, want_buf = wo.blend_md(outs, plan.batched_bboxes, N, x.shape, x.dtype, plan.weights)
    douts = [o.cuda() for o in outs]
    wts = torch.from_numpy(plan.weights).cuda()
    rcp = engine.exact_reciprocals(plan.weights)
    assert rcp is not None
    for flags in (0, TD_FLAG_FORCE_GENERIC):
        for use_rcp in (False, True):
            buf = torch.empty_like(x).cuda()
            got = engine.blend_multidiffusion(g, douts, N, C, g.tile_bs, wts, x.dtype, x_buffer=buf, flags=flags,
                                              rcp_weights=torch.from_numpy(rcp).cuda() if use_rcp else None)
            assert_bit_equal(got.cpu(), want, f"wrap MD {dn} {wrap} {shape} flags={flags} rcp={use_rcp}")
            assert_bit_equal(buf.cpu(), want_buf, "x_buffer")
        got = engine.blend_multidiffusion(g, douts, N, C, g.tile_bs, wts, x.dtype, flags=flags)
        assert_bit_equal(got.cpu(), want, "without x_buffer")


@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("wrap", WRAPS)
@pytest.mark.parametrize("shape", SHAPES)
def test_blend_mixture_bit_exact(dn, wrap, shape):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TD_FLAG_FORCE_GENERIC
    g, plan, x = _setup(shape, wrap, dn, gaussian=True, seed=3)
    N, C = x.shape[:2]
    outs = _tile_outs(plan, x, 4)
    want = wo.blend_mod(outs, plan.batched_bboxes, N, x.shape, x.dtype, plan.tile_weights, plan.rescale_factor)
    douts = [o.cuda() for o in outs]
    for flags in (0, TD_FLAG_FORCE_GENERIC):
        buf = torch.empty_like(x).cuda()
        got = engine.blend_mixture(g, douts, N, C, g.tile_bs, torch.from_numpy(plan.tile_weights).cuda(),
                                   torch.from_numpy(plan.rescale_factor).cuda(), buf, flags=flags)
        assert_bit_equal(got.cpu(), want, f"wrap MoD {dn} {wrap} {shape} flags={flags}")


def test_wide_panorama_blend_bit_exact():
    """A panorama-shaped latent wrapped in x only: 43 tile columns, the last ones crossing the seam."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    g, plan, x = _setup((1024, 128, 96, 96, 48, 8), wo.WRAP_X, "f16", seed=5)
    N, C = x.shape[:2]
    outs = _tile_outs(plan, x, 6)
    want, _ = wo.blend_md(outs, plan.batched_bboxes, N, x.shape, x.dtype, plan.weights)
    got = engine.blend_multidiffusion(g, [o.cuda() for o in outs], N, C, g.tile_bs, torch.from_numpy(plan.weights).cuda(), x.dtype)
    assert_bit_equal(got.cpu(), want, "panorama MD")
    assert_bit_equal(engine.scatter_tiles(g, x.cuda()).cpu(), wo.scatter(x, plan.bboxes), "panorama scatter")


@pytest.mark.parametrize("dn", list(DTYPES))
def test_tile_as_wide_as_the_canvas_reaches_a_vector_twice(dn):
    """A hand-made periodic plan whose tiles are as wide as the canvas but do not start at 0: the canvas vector holding a
    tile's origin also holds that tile's last columns, which arrive after the seam."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdGrid
    W, H, N, C = 64, 16, 2, 4
    g = TdGrid()
    g.W, g.H, g.tile_w, g.tile_h, g.overlap = W, H, W, H, 8
    g.rows, g.cols, g.num_tiles, g.num_batches, g.tile_bs = 1, 2, 2, 1, 2
    g.ys[0], g.xs[0], g.xs[1] = 0, 0, 21
    g.wrap = engine.WRAP_X
    bboxes = [(0, 0, W, H), (21, 0, W, H)]
    x = (torch.randn((N, C, H, W), generator=torch.Generator().manual_seed(14)) * 2).to(DTYPES[dn])
    assert_bit_equal(engine.scatter_tiles(g, x.cuda()).cpu(), wo.scatter(x, bboxes), "scatter")
    out = (torch.randn((2 * N, C, H, W), generator=torch.Generator().manual_seed(15))).to(x.dtype)
    weights = wo.weights(bboxes, W, H)
    want, want_buf = wo.blend_md([out], [bboxes], N, x.shape, x.dtype, weights)
    buf = torch.empty_like(x).cuda()
    got = engine.blend_multidiffusion(g, [out.cuda()], N, C, 2, torch.from_numpy(weights).cuda(), x.dtype, x_buffer=buf)
    assert_bit_equal(got.cpu(), want, "MD")
    assert_bit_equal(buf.cpu(), want_buf, "MD x_buffer")
    from oracle import tiling
    tw = tiling.gaussian_weights(W, H)
    gw = wo.weights(bboxes, W, H, tw)
    rs = (np.float32(1.0) / gw).astype(np.float32)
    want = wo.blend_mod([out], [bboxes], N, x.shape, x.dtype, tw, rs)
    got = engine.blend_mixture(g, [out.cuda()], N, C, 2, torch.from_numpy(tw).cuda(), torch.from_numpy(rs).cuda(), torch.empty_like(x).cuda())
    assert_bit_equal(got.cpu(), want, "MoD")


# ------------------------------------------------------------------------------------------------ delegates
GRID = dict(N=2, C=4, W=64, H=48, tw=24, th=16, ov=8, bs=3)
_BG, _FG = "Background", "Foreground"
REGIONS = [(True, 0.1, 0.2, 0.5, 0.4, "a cat", "", _BG, 0.2, -1),
           (True, 0.4, 0.3, 0.45, 0.6, "a dog", "", _FG, 0.3, 5)]


def _p():
    return types.SimpleNamespace(width=GRID["W"] * 8, height=GRID["H"] * 8, sampler_name="Euler a", disable_extra_networks=True)


def _sampler():
    return types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None,
                                                                      step=0))


@pytest.fixture
def shared():
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    state = types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1)
    host.use_shared(types.SimpleNamespace(state=state, sd_model=None))
    yield
    host.use_shared(None)


def _md_delegate(wrap, regions=False):
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion
    c = GRID
    d = MultiDiffusion(_p(), _sampler())
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"], wrap_x=bool(wrap & wo.WRAP_X), wrap_y=bool(wrap & wo.WRAP_Y))
    if regions:
        d.init_custom_bbox({i: row for i, row in enumerate(REGIONS)}, True, False)
    d.init_done()
    return d


@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_X | wo.WRAP_Y])
@pytest.mark.parametrize("dn", ["f16", "f32"])
def test_multidiffusion_delegate_matches_oracle(shared, wrap, dn):
    c = GRID
    d = _md_delegate(wrap)
    plan = wo.WrapPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], wrap)
    assert [(b.x, b.y, b.w, b.h) for bb in d.batched_bboxes for b in bb] == plan.bboxes
    x = (torch.randn((c["N"], c["C"], c["H"], c["W"]), generator=torch.Generator().manual_seed(7))).to(DTYPES[dn])
    for step in range(3):
        got = d.sample_one_step(x.cuda(), None, wo.blur_denoise, None)
        want, _ = wo.multidiffusion_step(x, plan, wo.blur_denoise)
        assert_bit_equal(got.cpu(), want, f"MD delegate wrap={wrap} step {step}")
        x = got.cpu().to(x.dtype)


def test_multidiffusion_delegate_with_regions(shared):
    """One BACKGROUND and one FOREGROUND region over a wrapped grid: the composite reads the accumulator the wrap blend wrote."""
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import BlendMode
    import oracle.synth as synth
    c = GRID
    wrap = wo.WRAP_X | wo.WRAP_Y
    d = _md_delegate(wrap, regions=True)
    plan = wo.WrapPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], wrap)
    x = (torch.randn((c["N"], c["C"], c["H"], c["W"]), generator=torch.Generator().manual_seed(8))).half()
    got = d.sample_one_step(x.cuda(), None, wo.blur_denoise, lambda xt, i, bb: synth.fake_region_denoise(xt, i))
    _, xbuf = wo.multidiffusion_step(x, plan, wo.blur_denoise)
    regions = []
    for i, b in enumerate(d.custom_bboxes):
        out = synth.fake_region_denoise(x[b.slicer], i)
        fg = b.blend_mode == BlendMode.FOREGROUND
        regions.append((b.x, b.y, b.w, b.h, int(fg), out, b.feather_mask.cpu().float().reshape(b.h, b.w) if fg else None))
    want = region_composite_reference(xbuf, d.weights.cpu().view(c["H"], c["W"]), regions)
    assert_bit_equal(got.cpu(), want, "MD wrap + regions")


def test_mixture_delegate_matches_oracle(shared):
    """Mixture of Diffusers through its model hook, with a spatial image cond (cropped by the scatter) on a wrapped grid."""
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, host
    c = GRID
    N = c["N"]
    wrap = wo.WRAP_X | wo.WRAP_Y
    d = MixtureOfDiffusers(_p(), _sampler())
    d.init_grid_bbox(c["tw"], c["th"], c["ov"], c["bs"], wrap_x=True, wrap_y=True)
    d.init_done()
    plan = wo.WrapPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], wrap, gaussian=True)
    icond = torch.randn((N, 5, c["H"], c["W"]), generator=torch.Generator().manual_seed(9)).half()
    seen = []

    def apply_model(x_tile, t, cond):
        seen.append(cond["c_concat"][0].cpu())
        return wo.blur_denoise(x_tile)
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="concat"))
    host.get_shared().sd_model = model
    d.hook()
    try:
        x = torch.randn((N, c["C"], c["H"], c["W"]), generator=torch.Generator().manual_seed(10)).half()
        cond = {"c_crossattn": [torch.zeros(N, 2, 4).cuda()], "c_concat": [icond.cuda()]}
        for step in range(2):
            seen.clear()
            got = model.apply_model(x.cuda(), torch.ones(N).cuda(), cond).clone()
            want = wo.mixture_step(x, plan, wo.blur_denoise)
            assert_bit_equal(got.cpu(), want, f"MoD delegate step {step}")
            assert_bit_equal(torch.cat(seen, 0), wo.scatter(icond, plan.bboxes), "spatial icond crops")
            x = got.cpu()
    finally:
        MixtureOfDiffusers.unhook()


def test_controlnet_hint_crop_is_modular(shared):
    """ControlNet hints live at 8x the latent: the wrapped plan scaled x8 crops them through the scatter kernel."""
    c = GRID
    d = _md_delegate(wo.WRAP_X)
    hint = torch.randn((1, 3, c["H"] * 8, c["W"] * 8), generator=torch.Generator().manual_seed(11)).half()
    got = d._crop_side_input(hint.cuda(), 8)
    want = wo.scatter(hint, [(x * 8, y * 8, w * 8, h * 8) for bb in d.batched_bboxes for (x, y, w, h) in ((b.x, b.y, b.w, b.h) for b in bb)])
    assert_bit_equal(got.cpu(), want, "hint crop")
    with pytest.raises(ValueError):
        d._crop_side_input(hint[:, :, :-8].cuda(), 8)


def test_get_noise_runs_the_wrapped_step(shared):
    """Noise inversion's get_noise goes through the same wrapped step."""
    from multidiffusion_upscaler_for_automatic1111_b200 import host
    c = GRID
    N = c["N"]
    d = _md_delegate(wo.WRAP_X | wo.WRAP_Y)
    plan = wo.WrapPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], wo.WRAP_X | wo.WRAP_Y)
    model = types.SimpleNamespace(apply_model=lambda x_tile, sigma, cond: wo.blur_denoise(x_tile), cond_stage_key="txt",
                                  model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.get_shared().sd_model = model
    x = torch.randn((N, c["C"], c["H"], c["W"]), generator=torch.Generator().manual_seed(12))
    cond = {"c_crossattn": [torch.zeros(N, 2, 4).cuda()], "c_concat": [torch.zeros(N, 5, 1, 1).cuda()]}
    got = d.get_noise(x.cuda(), torch.ones(N).cuda(), cond, 0)
    want, _ = wo.multidiffusion_step(x, plan, wo.blur_denoise)
    assert_bit_equal(got.cpu(), want, "get_noise")


def test_controlnet_hint_inside_the_step(shared):
    """The hint crops the ControlNet unit sees during a wrapped MultiDiffusion step are the modular crops of its hint."""
    c = GRID
    N = c["N"]
    d = _md_delegate(wo.WRAP_X | wo.WRAP_Y)
    hint = torch.randn((1, 3, c["H"] * 8, c["W"] * 8), generator=torch.Generator().manual_seed(16)).half()
    unit = types.SimpleNamespace(hint_cond=hint.cuda())
    d.init_controlnet(types.SimpleNamespace(latest_network=types.SimpleNamespace(control_params=[unit])), False)
    seen = []

    def repeat_func(x_tile, bboxes):
        seen.append(unit.hint_cond.cpu())
        return wo.blur_denoise(x_tile)
    x = torch.randn((N, c["C"], c["H"], c["W"]), generator=torch.Generator().manual_seed(17)).half()
    got = d.sample_one_step(x.cuda(), None, repeat_func, None)
    plan = wo.WrapPlan(c["W"], c["H"], c["tw"], c["th"], c["ov"], c["bs"], wo.WRAP_X | wo.WRAP_Y)
    assert_bit_equal(got.cpu(), wo.multidiffusion_step(x, plan, wo.blur_denoise)[0], "step with a ControlNet unit")
    for bbs, crops in zip(plan.batched_bboxes, seen):
        want = wo.scatter(hint, [(bx * 8, by * 8, bw * 8, bh * 8) for (bx, by, bw, bh) in bbs])
        want = want.repeat_interleave(N, dim=0) if d.is_kdiff else want.repeat([N * 2, 1, 1, 1])
        assert_bit_equal(crops, want, "hint crop of a tile batch")


def test_refusals(shared):
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion
    d = _md_delegate(wo.WRAP_X)
    with pytest.raises(NotImplementedError):
        d.init_tile_shard(None)
    df = DemoFusion.__new__(DemoFusion)
    df.method = "DemoFusion"
    with pytest.raises(NotImplementedError):
        df.init_grid_bbox(16, 16, 8, 4, wrap_x=True)


def test_step_commutes_with_a_roll():
    """The seam property.  On a plan whose stride divides the canvas (L = 512, tile 128, overlap 64: stride 64), rolling the
    latent by one stride and stepping equals stepping and rolling, up to the add order at the seam (fp32: 1e-6 relative).
    The bounded plan of the same shape does not have this property at the edges."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N, C, L = 1, 4, 512
    x = torch.randn((N, C, L, L), generator=torch.Generator().manual_seed(13)).cuda()

    def step(g, xx):
        tiles = engine.scatter_tiles(g, xx)
        outs = [wo.blur_denoise(tiles[b * g.tile_bs * N:min((b + 1) * g.tile_bs, g.num_tiles) * N]) for b in range(g.num_batches)]
        wts = torch.from_numpy(engine.grid_weights(g)).cuda()
        return engine.blend_multidiffusion(g, outs, N, C, g.tile_bs, wts, xx.dtype)

    for wrap, seamless in ((engine.WRAP_X | engine.WRAP_Y, True), (0, False)):
        g = engine.make_grid(L, L, 128, 128, 64, 8, wrap=wrap)
        a = step(g, torch.roll(x, (64, 64), (2, 3)))
        b = torch.roll(step(g, x), (64, 64), (2, 3))
        rel = ((a - b).abs().max() / b.abs().max()).item()
        if seamless:
            assert list(g.xs[:g.cols]) == list(range(0, L, 64))
            assert rel <= 1e-6, rel
        else:
            assert rel > 1e-2, rel


# ------------------------------------------------------------------------------------------------ tiled VAE
@pytest.fixture(scope="module")
def tv():
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return tilevae


def _hook(tv, net, tile, is_dec, fast, wrap):
    hook = tv.VAEHook(net, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=False)
    hook.wrap_x, hook.wrap_y = bool(wrap & wo.WRAP_X), bool(wrap & wo.WRAP_Y)
    return hook


@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_X | wo.WRAP_Y])
@pytest.mark.parametrize("bbox", [(-11, 24, -11, 24), (30, 63, 2, 37), (-5, 60, 20, 51), (0, 52, 0, 40)])
def test_modular_tile_load_both_backends(tv, wrap, bbox):
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine as ve
    z = torch.randn((2, 4, 40, 52), generator=torch.Generator().manual_seed(18)).half().cuda()
    want = wo.load_wrap(z, bbox)
    mb = ve.ModuleBackend.__new__(ve.ModuleBackend)
    mb.dtype, mb.device = torch.float16, z.device
    mod = mb.load_wrap(z, bbox)
    assert_bit_equal(mod.cpu(), want.cpu(), "module backend load")
    tc = ve.TensorCoreBackend.__new__(ve.TensorCoreBackend)
    tc.dtype, tc.device = torch.float16, z.device
    got = tc.load_wrap(z, bbox)
    assert got.shape == (2, bbox[3] - bbox[2], bbox[1] - bbox[0], 64)
    assert_bit_equal(got[..., :4].permute(0, 3, 1, 2).cpu(), want.cpu(), "channels-last load")
    assert not got[..., 4:].any()


# module backend (fp32 networks), held to the tolerance of the bounded fp32 decode / encode
@pytest.mark.parametrize("is_dec,fast,H,W,tile,batch", [(True, False, 40, 52, 16, 1), (True, True, 40, 52, 16, 1), (True, False, 40, 52, 16, 2),
                                                         (False, False, 200, 264, 64, 1), (False, True, 200, 264, 64, 1),
                                                         (True, False, 24, 24, 16, 1)])
@pytest.mark.parametrize("wrap", [wo.WRAP_X, wo.WRAP_X | wo.WRAP_Y])
def test_vae_wrap_module_backend_matches_oracle(tv, is_dec, fast, H, W, tile, batch, wrap):
    from oracle.make_golden import vae_case_inputs
    net, z = vae_case_inputs(is_dec, H, W)
    if batch == 2:
        z = torch.cat([z, z.flip(3)], dim=0)
    with torch.no_grad():
        want = wo.vae_tile_forward_wrap(net, z, tile, is_dec, fast, wrap)
    net_gpu, _ = vae_case_inputs(is_dec, H, W)
    net_gpu = net_gpu.cuda()
    net_gpu.original_forward = net_gpu.forward
    hook = _hook(tv, net_gpu, tile, is_dec, fast, wrap)
    with torch.no_grad():
        got = hook(z.cuda())
    assert hook.backend_name == "modules" and got.shape == want.shape
    assert tuple(net_gpu.last_z_shape) == tuple(z.shape)          # tiled, also below the tiny-input bound
    scale = max(1.0, want.abs().max().item())
    assert (got.cpu() - want).abs().max().item() <= 3e-4 * scale


def _sd_width_net(is_dec, seed):
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), seed)
    net.eval()
    net.original_forward = net.forward
    return net


@pytest.mark.parametrize("is_dec,fast,H,W,tile,batch", [(True, True, 40, 52, 16, 1), (True, False, 40, 52, 16, 1), (True, False, 40, 52, 16, 2),
                                                         (False, True, 200, 264, 64, 1), (False, False, 136, 200, 64, 1)])
def test_vae_wrap_tensor_core_backend_matches_oracle(tv, is_dec, fast, H, W, tile, batch):
    from oracle import synth
    wrap = wo.WRAP_X | wo.WRAP_Y
    z = synth.latent(5 if is_dec else 6, (batch, 4 if is_dec else 3, H, W), torch.float32)
    ref_net = _sd_width_net(is_dec, 3 if is_dec else 4).cuda()
    with torch.no_grad():
        want = wo.vae_tile_forward_wrap(ref_net, z.cuda(), tile, is_dec, fast, wrap).cpu()
    hook = _hook(tv, _sd_width_net(is_dec, 3 if is_dec else 4).cuda().half(), tile, is_dec, fast, wrap)
    with torch.no_grad():
        got = hook(z.cuda().half())
    assert hook.backend_name == "wgmma" and got.shape == want.shape
    diff = (got.cpu().float() - want).abs()
    scale = want.abs().max().item()
    assert diff.mean().item() <= 2e-3 * scale and diff.max().item() <= 3e-2 * scale, (diff.mean().item() / scale, diff.max().item() / scale)


def test_vae_wrap_decode_with_parking_is_bit_identical(tv):
    """Slow wrap decode with a forced GPU-residency budget: tiles wait in pinned host memory, same output bits."""
    from oracle import synth
    hook = _hook(tv, _sd_width_net(True, 3).cuda().half(), 8, True, False, wo.WRAP_X | wo.WRAP_Y)
    z = synth.latent(5, (1, 4, 40, 52), torch.float16).cuda()
    with torch.no_grad():
        hook.max_resident_bytes = None
        a = hook(z)
        assert sum(hook.last_park_stats["tiles_parked"].values()) == 0
        hook.max_resident_bytes = 0
        b = hook(z)
    torch.cuda.synchronize()
    assert sum(hook.last_park_stats["tiles_parked"].values()) > 0
    assert torch.equal(a, b)
