"""Parity tests proper: the sm_90a kernels, called through the C-ABI, against the oracle
and the reference-generated fixtures.  Bit-exact (integer/index work AND the fp blend:
the gather-form kernel reproduces the reference's rounding sequence)."""
import os
import types

import numpy as np
import pytest
import torch

from helpers import load_golden, DTYPES, assert_bit_equal, bits, sha
from oracle import blend, synth, tiling

pytestmark = pytest.mark.gpu

FORCE_GENERIC = 1
NO_TMA = 2
TMA = 4
PIPE = 8
NO_PDL = 32
ONE_PLANE = 64
ROWS = 0x400
# cp.async-staged (default), row-block bulk-copy form (opt-in, td_rows.cu), persistent pipelined cp.async,
# TMA-staged, register-staged, scalar kernels
ALL_PATHS = [0, NO_PDL, ROWS, ROWS | NO_PDL, ONE_PLANE, PIPE, TMA, NO_TMA, FORCE_GENERIC]


@pytest.fixture(scope="module")
def eng():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine


def _grid(eng, W, H, tw, th, ov, bs):
    return eng.make_grid(W, H, tw, th, ov, bs)


SCATTER_CASES = [  # N, C, W, H, tw, th, ov
    (2, 4, 64, 48, 16, 16, 8), (1, 4, 57, 43, 16, 16, 12), (2, 4, 128, 128, 96, 96, 48), (3, 5, 96, 64, 40, 24, 4),
    (2, 4, 512, 512, 96, 96, 48), (1, 9, 72, 72, 24, 16, 6), (2, 4, 100, 77, 32, 24, 8),
]


@pytest.mark.parametrize("case", SCATTER_CASES)
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("flags", ALL_PATHS)
def test_scatter_bit_exact(eng, case, dn, flags):
    N, C, W, H, tw, th, ov = case
    g = _grid(eng, W, H, tw, th, ov, 4)
    x = synth.latent(7, (N, C, H, W), DTYPES[dn])
    plan = tiling.GridPlan(W, H, tw, th, ov, 4, False)
    want = blend.scatter_tiles(x, plan.bboxes)
    got = eng.scatter_tiles(g, x.cuda(), flags=flags)
    assert_bit_equal(got, want, "scatter")
    # a sub-range of tiles (what one rank of a tile-sharded run scatters)
    lo, hi = g.num_tiles // 3, g.num_tiles - 1
    if hi > lo:
        part = eng.scatter_tiles(g, x.cuda(), tile_begin=lo, tile_end=hi, flags=flags)
        assert_bit_equal(part, want[lo * N:hi * N], "scatter range")


def _run_cuda_step(eng, method, x, W, H, tw, th, ov, bs, flags=0, one_batch=False, tile_dtype=None, use_rcp=False):
    """scatter -> fake UNet per batch (on the GPU) -> fused blend, through the engine wrappers."""
    N, C = x.shape[:2]
    g = _grid(eng, W, H, tw, th, ov, bs)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, method == "mod")
    xd = x.cuda()
    tiles = eng.scatter_tiles(g, xd, flags=flags)
    outs = []
    tile_bs = g.num_tiles if one_batch else g.tile_bs
    batches = [plan.bboxes] if one_batch else plan.batched_bboxes
    off = 0
    for bbs in batches:
        t = tiles[off * N:(off + len(bbs)) * N]
        o = synth.fake_denoise(t, bbs, N)
        if tile_dtype is not None:
            o = o.to(tile_dtype)
        outs.append(o)
        off += len(bbs)
    if method == "md":
        w = torch.from_numpy(plan.weights).cuda()
        xb = torch.empty_like(xd)
        rcp = torch.from_numpy(eng.exact_reciprocals(plan.weights)).cuda() if use_rcp else None
        out = eng.blend_multidiffusion(g, outs, N, C, tile_bs, w, xd.dtype, x_buffer=xb, flags=flags, rcp_weights=rcp)
        return out, xb, plan
    twt = torch.from_numpy(plan.tile_weights).cuda()
    rf = torch.from_numpy(plan.rescale_factor).cuda()
    xb = torch.empty_like(xd)
    eng.blend_mixture(g, outs, N, C, tile_bs, twt, rf, xb, flags=flags)
    return xb, xb, plan


def _oracle_step(method, x, plan, tile_dtype=None):
    N = x.shape[0]

    def den(t, bb):
        o = synth.fake_denoise(t, bb, N)
        return o if tile_dtype is None else o.to(tile_dtype)
    if method == "md":
        return blend.multidiffusion_step(x, plan.batched_bboxes, plan.weights, den)
    return blend.mixture_step(x, plan.batched_bboxes, plan.tile_weights, plan.rescale_factor, den)


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
@pytest.mark.parametrize("flags", ALL_PATHS)
def test_blend_small_matches_reference_fixtures(eng, golden_dir, method, dn, flags):
    g = load_golden(golden_dir, "blend_small")
    for name, (N, C, W, H, tw, th, ov, bs) in zip(g["names"], g["cases"]):
        x = synth.latent(synth.case_seed(str(name), dn), (int(N), int(C), int(H), int(W)), DTYPES[dn])
        out, _, _ = _run_cuda_step(eng, method, x, int(W), int(H), int(tw), int(th), int(ov), int(bs), flags=flags)
        key = f"{name}_{dn}_{method}"
        assert str(out.dtype) == str(g[key + "_dtype"]), key
        assert np.array_equal(bits(out), g[key]), f"{key}: CUDA output differs from the reference's"


@pytest.mark.parametrize("dn", ["f16", "bf16"])
def test_fast_exact_divide_is_ieee_on_its_domain(dn):
    """q = a*rcp; r = fma(-q, w, a); q += r*rcp  ==  IEEE a / w for EVERY 16-bit numerator and integer w <= 4096."""
    import ctypes
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    _cabi.check(_cabi.lib.td_debug_check_fast_div(_cabi.dtype_code(DTYPES[dn]), 4096, bad.data_ptr(), _cabi.current_stream_ptr()))
    torch.cuda.synchronize()
    assert int(bad.item()) == 0


@pytest.mark.parametrize("dn", ["f16", "bf16"])
@pytest.mark.parametrize("flags", [0, ROWS, PIPE, TMA, NO_TMA])
def test_blend_with_reciprocal_weights_matches_reference(eng, golden_dir, dn, flags):
    g = load_golden(golden_dir, "blend_small")
    for name, (N, C, W, H, tw, th, ov, bs) in zip(g["names"], g["cases"]):
        x = synth.latent(synth.case_seed(str(name), dn), (int(N), int(C), int(H), int(W)), DTYPES[dn])
        out, _, _ = _run_cuda_step(eng, "md", x, int(W), int(H), int(tw), int(th), int(ov), int(bs), flags=flags, use_rcp=True)
        assert np.array_equal(bits(out), g[f"{name}_{dn}_md"]), f"{name}: fast-divide output differs from the reference's"
    h = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
    idx = list(h["names"]).index("cfg2_ov48")
    N, C, W, H, tw, th, ov, bs = map(int, h["cases"][idx])
    x = synth.latent(synth.case_seed("cfg2_ov48", dn), (N, C, H, W), DTYPES[dn])
    out, _, _ = _run_cuda_step(eng, "md", x, W, H, tw, th, ov, bs, flags=flags, use_rcp=True)
    assert sha(out) == str(h[f"cfg2_ov48_{dn}_md"])


@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", list(DTYPES))
def test_blend_full_size_hash(eng, golden_dir, method, dn):
    """BASELINE configs at full size: sha256 of the output equals the reference's."""
    g = np.load(os.path.join(golden_dir, "blend_hashes.npz"))
    for name, (N, C, W, H, tw, th, ov, bs) in zip(g["names"], g["cases"]):
        key = f"{name}_{dn}_{method}"
        if key not in g.files:
            continue
        x = synth.latent(synth.case_seed(str(name), dn), (int(N), int(C), int(H), int(W)), DTYPES[dn])
        for one_batch in (False, True):
            out, _, _ = _run_cuda_step(eng, method, x, int(W), int(H), int(tw), int(th), int(ov), int(bs), one_batch=one_batch)
            assert sha(out) == str(g[key]), f"{key} one_batch={one_batch}"


@pytest.mark.parametrize("method", ["md", "mod"])
def test_blend_vs_oracle_edge_geometries(eng, method):
    cases = [  # N, C, W, H, tw, th, ov, bs
        (1, 4, 96, 96, 96, 96, 48, 4),      # single tile
        (2, 4, 40, 30, 96, 96, 48, 4),      # tile clamped to the canvas, overlap > tile
        (2, 4, 97, 96, 96, 96, 48, 4),      # dx = 1: almost fully overlapping tiles
        (1, 4, 200, 8, 16, 8, 12, 7),       # long thin canvas, many columns
        (2, 4, 8, 200, 8, 16, 12, 5),
        (1, 1, 104, 104, 24, 24, 20, 16),   # overlap 20 of 24: up to 36 tiles per pixel
        (2, 4, 768, 768, 128, 128, 64, 8),  # DemoFusion-sized window
    ]
    for (N, C, W, H, tw, th, ov, bs) in cases:
        for dn in ("f16", "f32"):
            x = synth.latent(W + H, (N, C, H, W), DTYPES[dn])
            for flags in ALL_PATHS:
                out, xb, plan = _run_cuda_step(eng, method, x, W, H, tw, th, ov, bs, flags=flags)
                want = _oracle_step(method, x, plan)
                assert_bit_equal(out, want, f"{method} {(N, C, W, H, tw, th, ov, bs)} {dn} flags={flags}")


def test_multidiffusion_x_buffer_is_the_unnormalised_accumulator(eng):
    x = synth.latent(2, (2, 4, 72, 72), torch.float16)
    out, xb, plan = _run_cuda_step(eng, "md", x, 72, 72, 24, 16, 6, 3)
    N = 2
    acc = torch.zeros_like(x)
    for bbs in plan.batched_bboxes:
        blend.accumulate_md(acc, synth.fake_denoise(blend.scatter_tiles(x, bbs), bbs, N), bbs, N)
    assert_bit_equal(xb, acc, "x_buffer")


@pytest.mark.parametrize("acc_dn,tile_dn", [("f16", "f32"), ("f32", "f16"), ("bf16", "f16")])
def test_mixed_tile_and_canvas_dtypes(eng, acc_dn, tile_dn):
    """UNet output dtype != latent dtype: `x_buffer += tile` rounds through the canvas dtype."""
    x = synth.latent(9, (2, 4, 64, 48), DTYPES[acc_dn])
    for method in ("md", "mod"):
        out, _, plan = _run_cuda_step(eng, method, x, 48, 64, 16, 16, 8, 4, tile_dtype=DTYPES[tile_dn])
        want = _oracle_step(method, x, plan, tile_dtype=DTYPES[tile_dn])
        assert_bit_equal(out, want, f"{method} acc={acc_dn} tile={tile_dn}")


# ---------------------------------------------------------------------------------------
# through the reference-facing classes
# ---------------------------------------------------------------------------------------
def _p(W, H):
    return types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name="Euler a")


class _KSampler:
    def __init__(self, fwd):
        inner = types.SimpleNamespace(forward=fwd)
        self.model_wrap_cfg = types.SimpleNamespace(inner_model=inner, image_cfg_scale=None, step=0)


@pytest.mark.parametrize("dn", list(DTYPES))
def test_multidiffusion_class_kdiff_forward(dn):
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion
    N, C, W, H, tw, th, ov, bs = 2, 4, 128, 128, 96, 96, 48, 4
    calls = []

    def unet(x_tile, sigma, cond=None):
        # tile-batch invariants the reference guarantees to the UNet
        n_rep = x_tile.shape[0] // N
        assert sigma.shape[0] == x_tile.shape[0]
        assert cond["c_crossattn"][0].shape[0] == x_tile.shape[0]
        assert cond["c_concat"][0].shape[0] == x_tile.shape[0]
        bbs = d.batched_bboxes[len(calls)]
        assert n_rep == len(bbs)
        calls.append(n_rep)
        return synth.fake_denoise(x_tile, bbs, N)

    d = MultiDiffusion(_p(W, H), _KSampler(unet))
    d.init_grid_bbox(tw, th, ov, bs)
    d.init_done()
    d.hook()
    x = synth.latent(21, (N, C, H, W), DTYPES[dn])
    cond = {"c_crossattn": [torch.zeros(N, 77, 16, device="cuda")], "c_concat": [torch.zeros(N, 5, 1, 1, device="cuda")]}
    sigma = torch.ones(N, device="cuda")
    out = d.sampler.model_wrap_cfg.inner_model.forward(x.cuda(), sigma, cond=cond)
    plan = tiling.GridPlan(W, H, tw, th, ov, bs, False)
    want = _oracle_step("md", x, plan)
    assert out.dtype == torch.float32
    assert_bit_equal(out, want, "MultiDiffusion.kdiff_forward")
    assert len(calls) == d.num_batches
    # second step reuses the persistent tile buffer and returns a FRESH tensor (multistep samplers keep old ones)
    calls.clear()
    out2 = d.sampler.model_wrap_cfg.inner_model.forward(x.cuda(), sigma, cond=cond)
    assert out2.data_ptr() != out.data_ptr()
    assert_bit_equal(out2, want, "second step")


@pytest.mark.parametrize("dn", ["f16", "f32"])
def test_mixture_class_apply_model(dn):
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, host
    N, C, W, H, tw, th, ov, bs = 2, 4, 128, 128, 96, 96, 48, 4
    it = {"i": 0}

    def apply_model(x_tile, t, c):
        bbs = d.batched_bboxes[it["i"]]
        it["i"] += 1
        assert t.shape[0] == x_tile.shape[0] and c["c_crossattn"][0].shape[0] == x_tile.shape[0]
        assert c["c_concat"][0].shape == (x_tile.shape[0], 5, th, tw)  # img2img: spatial icond cropped per tile
        return synth.fake_denoise(x_tile, bbs, N)

    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt",
                                  model=types.SimpleNamespace(conditioning_key="hybrid"))
    host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1),
                                          sd_model=model))
    try:
        d = MixtureOfDiffusers(_p(W, H), _KSampler(None))
        d.init_grid_bbox(tw, th, ov, bs)
        d.init_done()
        d.hook()
        x = synth.latent(22, (N, C, H, W), DTYPES[dn])
        cond = {"c_crossattn": [torch.zeros(N, 77, 16, device="cuda")],
                "c_concat": [torch.zeros(N, 5, H, W, device="cuda", dtype=DTYPES[dn])]}
        out = model.apply_model(x.cuda(), torch.ones(N, device="cuda"), cond)
        plan = tiling.GridPlan(W, H, tw, th, ov, bs, True)
        want = _oracle_step("mod", x, plan)
        assert out.dtype == DTYPES[dn] and out.data_ptr() == d.x_buffer.data_ptr()
        assert_bit_equal(out, want, "MixtureOfDiffusers.apply_model_hijack")
        MixtureOfDiffusers.unhook()
        assert model.apply_model is apply_model
    finally:
        host.use_shared(None)


def test_interrupt_returns_input_untouched():
    from multidiffusion_upscaler_for_automatic1111_b200 import MultiDiffusion, host
    st = types.SimpleNamespace(interrupted=True, sampling_step=0, sampling_steps=1)
    host.use_shared(types.SimpleNamespace(state=st, sd_model=None))
    try:
        d = MultiDiffusion(_p(64, 64), _KSampler(lambda x, s, cond=None: x))
        d.init_grid_bbox(16, 16, 4, 4)
        d.init_done()
        x = synth.latent(1, (2, 4, 64, 64), torch.float16).cuda()
        assert d.sample_one_step(x, None, lambda t, b: t, None) is x
    finally:
        host.use_shared(None)


def test_size_independent_properties_at_cfg1(eng):
    """1024x1024 latent (BASELINE cfg1 literal reading): constant field is a fixed point of
    MultiDiffusion, and the blend is linear in the tile outputs where accumulation is exact (fp32)."""
    N, C, W, H = 2, 4, 1024, 1024
    g = _grid(eng, W, H, 96, 96, 4, 8)
    plan_w = torch.from_numpy(eng.grid_weights(g)).cuda()
    x = torch.full((N, C, H, W), 0.75, dtype=torch.float16, device="cuda")
    tiles = eng.scatter_tiles(g, x)
    out = eng.blend_multidiffusion(g, [tiles], N, C, g.num_tiles, plan_w, x.dtype)
    assert torch.equal(out, x.float())  # identity denoiser: every pixel is k*0.75/k
    a = synth.latent(3, (N, C, H, W), torch.float32).cuda()
    b = synth.latent(4, (N, C, H, W), torch.float32).cuda()
    ta, tb = eng.scatter_tiles(g, a).clone(), eng.scatter_tiles(g, b).clone()
    oa = eng.blend_multidiffusion(g, [ta], N, C, g.num_tiles, plan_w, torch.float32)
    ob = eng.blend_multidiffusion(g, [tb], N, C, g.num_tiles, plan_w, torch.float32)
    oab = eng.blend_multidiffusion(g, [ta + tb], N, C, g.num_tiles, plan_w, torch.float32)
    assert torch.allclose(oab, oa + ob, rtol=0, atol=1e-5)
    # identity denoiser reproduces the input exactly for values with short significands
    assert torch.equal(oa, a)


def test_bad_arguments_return_status_not_crash(eng):
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    g = _grid(eng, 64, 64, 16, 16, 4, 4)
    x = torch.zeros(2, 4, 64, 64, device="cuda", dtype=torch.float16)
    with pytest.raises(_cabi.TdError) as e:
        eng.scatter_tiles(g, x, tile_begin=5, tile_end=g.num_tiles + 1)
    assert e.value.status == _cabi.TD_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        eng.scatter_tiles(g, torch.zeros(2, 4, 32, 64, device="cuda"))
    w = torch.ones(64, 64, device="cuda")
    tiles = eng.scatter_tiles(g, x)
    with pytest.raises(ValueError):
        eng.blend_multidiffusion(g, [tiles[:-2]], 2, 4, g.num_tiles, w, x.dtype)
    with pytest.raises((_cabi.TdError, ValueError)):
        eng.blend_multidiffusion(g, [tiles], 2, 4, g.num_tiles - 1, w, x.dtype)  # table does not cover the tiles


@pytest.mark.parametrize("graph,wrap", [(False, 0), (True, 0), (False, 3), (True, 3)], ids=["False", "True", "False-wrap", "True-wrap"])
def test_dependent_launch_chain_keeps_stream_order(eng, graph, wrap):
    """The default kernels are launched with programmatic dependent launch.  A chain in which every kernel consumes
    what its direct predecessor wrote (scatter reads the canvas the blend just wrote, the blend reads the tiles the
    scatter just wrote, and overwrites the canvas the scatter just read) must equal the plainly serialised run bit for
    bit, eagerly and when replayed from a CUDA graph, on a bounded and on a periodic plan (wrap = 3: x and y, the
    td_wrap.cu kernels, whose blends load their origins and release the next launch before waiting), in the vector
    and in the generic forms."""
    N, C, W, H, tw, th, ov, bs = 2, 4, 512, 512, 96, 96, 48, 4
    g = eng.make_grid(W, H, tw, th, ov, bs, wrap=wrap)
    if wrap:
        import wrap_oracle as wo
        plan = wo.WrapPlan(W, H, tw, th, ov, bs, wrap, gaussian=True)
        assert list(g.xs[:g.cols]) == plan.xs and list(g.ys[:g.rows]) == plan.ys
    else:
        plan = tiling.GridPlan(W, H, tw, th, ov, bs, True)
    twt = torch.from_numpy(plan.tile_weights).cuda()
    rf = torch.from_numpy(plan.rescale_factor).cuda()
    x0 = synth.latent(31, (N, C, H, W), torch.float16).cuda()
    iters = 24

    def chain(flags):
        xb = x0.clone()
        tiles = torch.empty((g.num_tiles * N, C, th, tw), dtype=torch.float16, device="cuda")
        # one batch holding every tile: the blend reads the scatter's output buffer in place
        def run():
            for _ in range(iters):
                eng.scatter_tiles(g, xb, out=tiles, flags=flags)
                eng.blend_mixture(g, [tiles], N, C, g.num_tiles, twt, rf, xb, flags=flags)
        if not graph:
            run()
        else:
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                run()                                   # warm-up outside capture (sets kernel attributes)
                xb.copy_(x0)
                cg = torch.cuda.CUDAGraph()
                with torch.cuda.graph(cg, stream=st):
                    run()
                cg.replay()
            torch.cuda.current_stream().wait_stream(st)
        torch.cuda.synchronize()
        return xb.clone()

    for form in (0, FORCE_GENERIC):
        want = chain(form | NO_PDL)
        got = chain(form)
        assert torch.isfinite(want.float()).all()
        assert_bit_equal(got, want.cpu(), f"PDL chain wrap={wrap} flags={form}")
