"""Tiled-VAE inpainting on the GPU: `td_vae_active_tiles` against the numpy rule, and `VAEHook.set_inpaint_mask` against the
unmasked decode -- bit-identical on every rectangle a pass runs, the fill (or zeros) on every rectangle it skips."""
import socket

import numpy as np
import pytest
import torch

from helpers import assert_bit_equal
from test_vae_inpaint_plan import active_rule, decoder_rects

pytestmark = pytest.mark.gpu

DTS = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}


@pytest.fixture(scope="module")
def m():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine, host, tilevae, vae_engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _cabi, engine, tilevae, vae_engine, host


def _not_one(dtype):
    """Values that are not 1 in `dtype`: its neighbours of 1.0, +-0, +-inf, NaN and -1."""
    ib = torch.int32 if dtype == torch.float32 else torch.int16
    one = torch.ones(1, dtype=dtype).view(ib)
    near = [(one + 1).view(dtype).item(), (one - 1).view(dtype).item()]
    return near + [0.0, -0.0, float("inf"), float("-inf"), float("nan"), -1.0]


def _check_kernel(m, mask, rects, what):
    got = m[1].vae_active_tiles(mask, rects)
    want = active_rule(mask.float().cpu().numpy(), rects)
    assert (got == want).all(), f"{what}: kernel {np.flatnonzero(got)} vs rule {np.flatnonzero(want)}"
    return got


# ------------------------------------------------------------------------------------------ td_vae_active_tiles
@pytest.mark.parametrize("dt", list(DTS))
def test_active_tiles_on_the_cfg4_split(m, dt):
    """8192 x 8192 image, 121 output rectangles: all keep, all inpaint, a 1024^2 square in the middle, and one element that
    is not 1 at a corner or an edge of every fifth rectangle (values next to 1, +-0, +-inf, NaN)."""
    rects = decoder_rects(1024, 1024, 96)
    assert len(rects) == 121
    mask = torch.ones(8192, 8192, dtype=DTS[dt], device="cuda")
    assert not _check_kernel(m, mask, rects, "all keep").any()
    assert _check_kernel(m, torch.zeros_like(mask), rects, "all inpaint").all()
    sq = mask.clone()
    sq[3584:4608, 3584:4608] = 0.25
    assert 0 < _check_kernel(m, sq, rects, "square").sum() < 121
    vals = _not_one(DTS[dt])
    for t in range(0, 121, 5):
        x1, x2, y1, y2 = rects[t]
        y, x = [(y1, x1), (y1, x2 - 1), (y2 - 1, x1), (y2 - 1, x2 - 1), (y1, (x1 + x2) // 2), ((y1 + y2) // 2, x1)][t % 6]
        mask[y, x] = vals[t % len(vals)]
    got = _check_kernel(m, mask, rects, "spots")
    assert got.sum() == len(range(0, 121, 5))


@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "misaligned"])
def test_active_tiles_on_ragged_rectangles(m, dt, planes, offset):
    """Odd sizes, rectangles of width 1 .. 80 at every alignment, the mask pointer off a 16-byte boundary: every row segment
    has a ragged head, body and tail somewhere.  One element that is not 1 per trial, in any plane."""
    H, W = 203, 301
    rng = np.random.default_rng(planes * 10 + offset)
    rects = []
    for _ in range(300):
        x1, y1 = int(rng.integers(0, W)), int(rng.integers(0, H))
        rects.append([x1, x1 + int(rng.integers(1, min(81, W - x1 + 1))), y1, y1 + int(rng.integers(1, min(40, H - y1 + 1)))])
    buf = torch.ones(planes * H * W + offset, dtype=DTS[dt], device="cuda")
    mask = buf[offset:].view(planes, H, W)
    assert (mask.data_ptr() % 16 != 0) == bool(offset)
    vals = _not_one(DTS[dt])
    assert not _check_kernel(m, mask, rects, "all keep").any()
    for trial in range(40):
        mask.fill_(1)
        p, y, x = int(rng.integers(0, planes)), int(rng.integers(0, H)), int(rng.integers(0, W))
        mask[p, y, x] = vals[trial % len(vals)]
        _check_kernel(m, mask, rects, f"trial {trial} at ({p}, {y}, {x})")
    # the whole canvas as one rectangle and a sparse random mask
    mask.fill_(1)
    mask.view(-1)[torch.from_numpy(rng.integers(0, planes * H * W, 50)).cuda()] = 0.5
    _check_kernel(m, mask, rects + [[0, W, 0, H]], "sparse")


def test_active_tiles_past_2_31_elements(m):
    """fp16 [2, 32800, 32800] (2^31 + 3.8e6 elements, 4.3 GB): the only element that is not 1 lies past element 2^31."""
    P, H, W = 2, 32800, 32800
    mask = torch.ones(P, H, W, dtype=torch.float16, device="cuda")
    mask[1, H - 1, W - 3] = 0.0
    assert (P - 1) * H * W + (H - 1) * W + W - 3 > 2 ** 31
    rects = [[0, W, 0, H], [W - 8, W, H - 8, H], [0, 8, 0, 8], [W - 2, W, H - 2, H], [W - 3, W - 2, H - 1, H]]
    got = m[1].vae_active_tiles(mask, rects)
    assert got.tolist() == [True, True, False, False, True]
    del mask
    torch.cuda.empty_cache()


def test_active_tiles_refusals_leave_the_output_untouched(m):
    cabi = m[0]
    import ctypes
    mask = torch.ones(64, 64, dtype=torch.float16, device="cuda")
    out = torch.full((4,), 0xAB, dtype=torch.uint8, device="cuda")

    def call(ptr=mask.data_ptr(), planes=1, H=64, W=64, dtype=cabi.TD_F16, rects=((0, 8, 0, 8),) * 4, outp=out.data_ptr()):
        r = np.ascontiguousarray(np.asarray(rects, dtype=np.int32).reshape(-1, 4))
        return cabi.lib.td_vae_active_tiles(ptr, planes, H, W, dtype, r.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(r),
                                            outp, cabi.current_stream_ptr())
    for kw, status in [(dict(ptr=None), cabi.TD_ERR_INVALID_ARG), (dict(ptr=mask.data_ptr() + 1), cabi.TD_ERR_INVALID_ARG),
                       (dict(ptr=mask.data_ptr() + 2, dtype=cabi.TD_F32), cabi.TD_ERR_INVALID_ARG),
                       (dict(planes=0), cabi.TD_ERR_INVALID_ARG), (dict(dtype=5), cabi.TD_ERR_INVALID_ARG),
                       (dict(rects=((0, 8, 0, 8),) * 3 + ((8, 8, 0, 8),)), cabi.TD_ERR_INVALID_ARG),
                       (dict(rects=((0, 8, 0, 8),) * 3 + ((60, 65, 0, 8),)), cabi.TD_ERR_INVALID_ARG),
                       (dict(H=0), cabi.TD_ERR_INVALID_ARG), (dict(planes=2 ** 16, H=2 ** 15 + 1), cabi.TD_ERR_UNSUPPORTED)]:
        assert call(**kw) == status, kw
        torch.cuda.synchronize()
        assert (out == 0xAB).all(), kw
    assert call() == cabi.TD_OK
    torch.cuda.synchronize()
    assert out.tolist() == [0, 0, 0, 0]


# ------------------------------------------------------------------------------------------ VAEHook
H, W, TILE = 40, 52, 8            # z [N, 4, 40, 52], tile 8: 12 tiles of a 320 x 416 image
_NETS = {}


def _hook(m, dtype):
    from oracle import ldm_vae
    if dtype not in _NETS:
        net = ldm_vae.seeded_init(ldm_vae.Decoder(), 3).eval()      # SD width
        net.original_forward = net.forward
        _NETS[dtype] = net.cuda().to(dtype)
    return m[2].VAEHook(_NETS[dtype], TILE, True, fast_decoder=True, fast_encoder=True, color_fix=False)


def _input(N, dtype, seed):
    from oracle import synth
    x = synth.latent(seed, (N, 4, H, W), torch.float32)
    x[N // 2] *= 3.0
    return x.to("cuda", dtype)


def _masks(N, dtype):
    """Per-image image-space masks: a blurred square reaching a few tiles, a thin vertical stroke, and (last image) keep all."""
    mk = torch.ones(N, 1, 8 * H, 8 * W, dtype=torch.float32)
    mk[0, 0, 40:90, 60:100] = 0.0
    mk[0, 0, 38:92, 58:102] = torch.where(mk[0, 0, 38:92, 58:102] == 1, torch.tensor(0.96), mk[0, 0, 38:92, 58:102])
    if N > 2:
        mk[1, 0, 150:300, 250:252] = 0.5
    return mk.to("cuda", dtype)


def _decode(hook, z, k=None, wrap=False, mask=None, fill=None):
    hook.images_per_pass = k
    hook.wrap_x = hook.wrap_y = wrap
    hook.set_inpaint_mask(mask, fill)
    try:
        with torch.no_grad():
            out = hook(z)
        torch.cuda.synchronize()
    finally:
        hook.set_inpaint_mask(None)
    return out, dict(hook.last_park_stats)


def _check_contract(got, want, fill, mask, rects, stats, what):
    """Per pass: the rectangles any image of the pass reaches are the unmasked bits, the others the fill (zeros)."""
    N, k = got.shape[0], stats["images_per_pass"]
    mk = mask.float().cpu().numpy()
    run = skipped = 0
    for s in range(0, N, k):
        imgs = range(s, min(s + k, N))
        active = np.any([active_rule(mk[n if mk.shape[0] > 1 else 0], rects) for n in imgs], axis=0)
        run, skipped = run + int(active.sum()), skipped + int((~active).sum())
        for n in imgs:
            for t, (x1, x2, y1, y2) in enumerate(rects):
                region = (n, slice(None), slice(y1, y2), slice(x1, x2))
                if active[t]:
                    assert_bit_equal(got[region], want[region], f"{what}: image {n} tile {t} (run)")
                else:
                    ref = torch.zeros_like(got[region]) if fill is None else fill[(n if fill.shape[0] > 1 else 0,) + region[1:]]
                    assert_bit_equal(got[region], ref, f"{what}: image {n} tile {t} (skipped)")
    assert (stats["tiles_run"], stats["tiles_skipped"]) == (run, skipped), (stats, run, skipped)
    assert 0 < run and 0 < skipped, what


HOOK_CASES = {     # net dtype, images_per_pass, wrap, mask dtype, fill form
    "f16_k1": ("f16", 1, False, torch.float32, "per_image"),
    "f16_auto": ("f16", None, False, torch.float16, "per_image"),
    "bf16_auto": ("bf16", None, False, torch.bfloat16, "zeros"),
    "bf16_k1_wrapped": ("bf16", 1, True, torch.float32, "broadcast"),
    "f16_auto_wrapped": ("f16", None, True, torch.float16, "per_image"),
    "f32_modules": ("f32", None, False, torch.float16, "per_image"),
    "f32_modules_wrapped": ("f32", None, True, torch.float32, "broadcast"),
}


@pytest.mark.parametrize("case", list(HOOK_CASES))
def test_masked_decode_is_the_unmasked_decode_on_the_tiles_it_runs(m, case):
    dt, k, wrap, mdt, fill_form = HOOK_CASES[case]
    dtype, N = DTS[dt], 3
    hook = _hook(m, dtype)
    z = _input(N, dtype, 31)
    want, st = _decode(hook, z, k, wrap)
    assert hook.backend_name == ("modules" if dt == "f32" else "wgmma")
    rects = hook.split_tiles(H, W)[1]          # 12 tiles bounded, 35 wrapped
    assert st["tiles_run"] == len(rects) * -(-N // st["images_per_pass"]) and st["tiles_skipped"] == 0, st
    mask = _masks(N, mdt)
    g = torch.Generator(device="cuda").manual_seed(5)
    fill = None if fill_form == "zeros" else \
        (torch.rand(N if fill_form == "per_image" else 1, 3, 8 * H, 8 * W, generator=g, device="cuda") * 2 - 1).to(dtype)
    got, st = _decode(hook, z, k, wrap, mask, fill)
    assert st["images_per_pass"] == (N if k is None else k), st
    _check_contract(got, want, fill, mask, rects, st, case)


def test_a_keep_all_mask_runs_no_tile_and_returns_the_fill(m):
    tv, ve = m[2], m[3]
    hook = _hook(m, torch.float16)
    z = _input(2, torch.float16, 41)
    fill = (torch.rand(1, 3, 8 * H, 8 * W, device="cuda") * 2 - 1).half()
    convs = {"estimate": 0, "tiles": 0}
    in_est = [False]
    real_conv, real_est = ve.TensorCoreBackend.conv, ve.Executor.estimate

    def conv(self, *a, **kw):
        convs["estimate" if in_est[0] else "tiles"] += 1
        return real_conv(self, *a, **kw)

    def estimate(self, *a, **kw):
        in_est[0] = True
        try:
            return real_est(self, *a, **kw)
        finally:
            in_est[0] = False
    ve.TensorCoreBackend.conv, ve.Executor.estimate = conv, estimate
    try:
        _decode(hook, z)
        assert convs["tiles"] > 0 and convs["estimate"] > 0, convs        # the spy sees the tiles' convolutions
        convs.update(estimate=0, tiles=0)
        got, st = _decode(hook, z, mask=torch.ones(8 * H, 8 * W, device="cuda"), fill=fill)
    finally:
        ve.TensorCoreBackend.conv, ve.Executor.estimate = real_conv, real_est
    assert convs["tiles"] == 0 and convs["estimate"] > 0, convs
    assert st["tiles_run"] == 0 and st["tiles_skipped"] == 12 * -(-2 // st["images_per_pass"]), st
    for n in range(2):
        assert_bit_equal(got[n:n + 1], fill, f"image {n}")


def test_an_image_whose_estimate_met_a_nan_runs_all_its_tiles(m, capsys):
    """Built as in the batched-pass test: an inf in image 1's latent makes the fast-mode estimate meet a NaN (the estimator
    input is standardised over the batch, so every image's may), and such an image runs in slow mode with every tile
    although its mask keeps everything; an image whose estimate held would run none.  Each image then runs alone and reports
    its NaN estimate, and the NaN check of the result still refuses the call."""
    hook = _hook(m, torch.float16)
    N = 3
    z = _input(N, torch.float16, 8)
    z[1, :, 3, 5] = float("inf")
    for k in (1, None):
        hook.images_per_pass = k
        hook.set_inpaint_mask(torch.ones(N, 1, 8 * H, 8 * W, device="cuda"))
        capsys.readouterr()
        try:
            with pytest.raises(RuntimeError, match="NaN"):
                with torch.no_grad():
                    hook(z)
        finally:
            hook.set_inpaint_mask(None)
        slow = capsys.readouterr().out.count("Nan detected in fast mode estimation")
        st = hook.last_park_stats
        assert slow >= 1 and st["tiles_run"] == 12 * slow and st["tiles_skipped"] == 12 * (N - slow), (k, slow, st)


def test_mismatched_mask_or_fill_is_refused_before_any_tile(m):
    ve = m[3]
    hook = _hook(m, torch.float16)
    z = _input(3, torch.float16, 2)
    img = (8 * H, 8 * W)
    bad = [dict(mask=torch.ones(2, 1, *img, device="cuda")), dict(mask=torch.ones(img[0], img[1] - 8, device="cuda")),
           dict(mask=torch.ones(*img, device="cuda"), fill=torch.zeros(1, 3, *img, device="cuda")),             # fp32 fill, fp16 net
           dict(mask=torch.ones(*img, device="cuda"), fill=torch.zeros(2, 3, *img, device="cuda").half()),
           dict(mask=torch.ones(*img, device="cuda"), fill=torch.zeros(3, 4, *img, device="cuda").half())]
    runs = [0]
    real = ve.Executor.run

    def run(self, *a, **kw):
        runs[0] += 1
        return real(self, *a, **kw)
    ve.Executor.run = run
    try:
        for kw in bad:
            hook.set_inpaint_mask(kw["mask"], kw.get("fill"))
            with pytest.raises(ValueError):
                with torch.no_grad():
                    hook(z)
    finally:
        ve.Executor.run = real
        hook.set_inpaint_mask(None)
    assert runs[0] == 0


def test_masked_decode_on_a_one_rank_nccl_group(m):
    import torch.distributed as dist
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        hook = _hook(m, torch.float16)
        hook.init_tile_shard(None)
        N = 3
        z = _input(N, torch.float16, 13)
        want, _ = _decode(hook, z)
        mask = _masks(N, torch.float16)
        fill = (torch.rand(N, 3, 8 * H, 8 * W, device="cuda") * 2 - 1).half()
        got, st = _decode(hook, z, mask=mask, fill=fill)
        rects = hook.split_tiles(H, W)[1]
        _check_contract(got, want, fill, mask, rects, st, "one-rank shard")
        # the exchange of the tiles a pass ran: one rank owns them all, so the gather leaves the canvas as it is
        active = np.flatnonzero(active_rule(mask.float().cpu().numpy()[0], rects)).tolist()
        out = got.clone()
        hook._shard_world, hook._shard_rank = 1, 0
        hook._exchange_regions(out, rects, [(slice(0, 1), active), (slice(1, N), list(range(len(rects))))])
        torch.cuda.synchronize()
        assert_bit_equal(out, got, "exchange")
    finally:
        dist.destroy_process_group()
