"""Tiled VAE with a GPU-memory budget: tiles that do not fit at a GroupNorm barrier wait in pinned host memory.  Parking
is a copy, so the output must be bit-identical to the run that keeps every tile on the device."""
import pytest
import torch

from helpers import assert_bit_equal

pytestmark = pytest.mark.gpu

DEC = (40, 52, 8)        # z [1, 4, 40, 52], tile 8: 12 tiles
ENC = (200, 264, 48)     # image [1, 3, 200, 264], tile 48: 15 tiles


@pytest.fixture(scope="module")
def mods():
    from multidiffusion_upscaler_for_automatic1111_b200 import host, tilevae, vae_engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return tilevae, vae_engine, host


def _net(is_dec, dtype):
    from oracle import ldm_vae
    net = ldm_vae.seeded_init((ldm_vae.Decoder if is_dec else ldm_vae.Encoder)(), 3 if is_dec else 4)
    net.eval()
    net.original_forward = net.forward
    return net.cuda().to(dtype)


def _case(mods, is_dec, dtype, fast=False, color_fix=False, batch=1):
    from oracle import synth
    tv, ve, _ = mods
    H, W, tile = DEC if is_dec else ENC
    net = _net(is_dec, dtype)
    x = synth.latent(5 if is_dec else 6, (batch, 4 if is_dec else 3, H, W), torch.float32).to("cuda", dtype)
    hook = tv.VAEHook(net, tile, is_dec, fast_decoder=fast, fast_encoder=fast, color_fix=color_fix)
    return hook, x


def _barrier_peak(ve, hook, x):
    """Predicted bytes of all tiles at the worst barrier site (per image on the tensor cores, whole batch on modules)."""
    prog = ve.compile_program(hook.net, hook.is_decoder)
    dtype = next(hook.net.parameters()).dtype
    backend = ve.pick_backend(prog, x.device, dtype).name
    ib, _ = hook.split_tiles(x.shape[2], x.shape[3])
    fps = [ve.tile_footprint(prog, backend, dtype, b[3] - b[2], b[1] - b[0], x.shape[0]) for b in ib]
    if hook.fast_mode:       # color fix: the sites from the first down-sampling on stay barriers
        sites = [op.site for i, op in enumerate(prog.ops) if isinstance(op, ve.Norm) and i >= prog.first_resample]
    else:
        sites = list(range(prog.num_sites))
    return max(sum(f.held(s) for f in fps) for s in sites)


def _run(hook, x, budget):
    hook.max_resident_bytes = budget
    with torch.no_grad():
        out = hook(x)
    torch.cuda.synchronize()
    return out, dict(hook.last_park_stats)


CASES = {
    "f16_slow_decode": dict(is_dec=True, dtype=torch.float16),
    "f16_slow_encode": dict(is_dec=False, dtype=torch.float16),
    "f16_fast_encode_color_fix": dict(is_dec=False, dtype=torch.float16, fast=True, color_fix=True),
    "f32_slow_decode_modules": dict(is_dec=True, dtype=torch.float32),
    "f16_slow_decode_batch2": dict(is_dec=True, dtype=torch.float16, batch=2),
    "f32_slow_decode_batch2_modules": dict(is_dec=True, dtype=torch.float32, batch=2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parked_runs_are_bit_identical(mods, name):
    tv, ve, _ = mods
    hook, x = _case(mods, **CASES[name])
    want, st = _run(hook, x, None)
    assert hook.backend_name == ("modules" if x.dtype == torch.float32 else "wgmma")
    assert st["tiles_parked"] == {} and st["d2h_bytes"] == 0 and st["host_bytes"] == 0
    again, _ = _run(hook, x, None)
    assert_bit_equal(again, want, f"{name}: two unbounded runs")
    peak = _barrier_peak(ve, hook, x)
    for budget in (peak // 3, 0):
        got, st = _run(hook, x, budget)
        assert_bit_equal(got, want, f"{name}: budget {budget} of {peak}")
        assert sum(st["tiles_parked"].values()) > 0 and st["d2h_bytes"] > 0 and st["h2d_bytes"] > 0 and st["host_bytes"] > 0
        assert st["budget"] == budget
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["wgmma", "modules"])
@pytest.mark.parametrize("is_dec", [True, False], ids=["decoder", "encoder"])
def test_predicted_bytes_match_the_tensors(mods, dtype, is_dec):
    tv, ve, _ = mods
    hook, x = _case(mods, is_dec, dtype)
    prog = ve.compile_program(hook.net, is_dec)
    backend = ve.pick_backend(prog, x.device, dtype).name
    ib, _ = hook.split_tiles(x.shape[2], x.shape[3])
    fps = [ve.tile_footprint(prog, backend, dtype, b[3] - b[2], b[1] - b[0], x.shape[0]) for b in ib]
    seen = []
    real = ve.Executor.run

    def spy(self, st, stop=None):
        op = real(self, st, stop)
        if op is not None:
            nb = lambda t: t.numel() * t.element_size()
            seen.append((op.site, nb(st.act), 0 if st.skip is None or st.skip is st.act else nb(st.skip)))
        return op
    ve.Executor.run = spy
    try:
        _run(hook, x, None)
    finally:
        ve.Executor.run = real
    n = len(ib)
    assert len(seen) == n * prog.num_sites
    for r in range(prog.num_sites):
        order = range(n) if r % 2 == 0 else range(n - 1, -1, -1)
        for k, i in enumerate(order):
            site, act, skip = seen[r * n + k]
            assert site == r
            assert (act, skip) == (fps[i].act[site], fps[i].skip[site]), f"tile {i} site {site}"


def test_memory_rise_stays_within_budget_and_reserve(mods):
    tv, ve, _ = mods
    hook, x = _case(mods, True, torch.float16)
    _run(hook, x, None)                     # weights packed, kernels loaded
    budget = _barrier_peak(ve, hook, x) // 3
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out, st = _run(hook, x, budget)
    rise = torch.cuda.max_memory_allocated() - base
    assert sum(st["tiles_parked"].values()) > 0
    allowance = st["budget"] + st["reserve"] + out.numel() * out.element_size() + (1 << 20)
    assert rise <= allowance, (rise, st)


def test_default_budget_parks_nothing(mods):
    for kw in (dict(is_dec=True, dtype=torch.float16), dict(is_dec=False, dtype=torch.float32)):
        hook, x = _case(mods, **kw)
        _, st = _run(hook, x, None)
        assert st["budget"] > 0
        assert st["tiles_parked"] == {} and st["d2h_bytes"] == 0 and st["h2d_bytes"] == 0 and st["host_bytes"] == 0


def test_interrupt_in_a_parked_round_returns_the_partial_result(mods):
    tv, ve, host = mods
    hook, x = _case(mods, True, torch.float16)
    want, _ = _run(hook, x, None)
    backend_cls = ve.TensorCoreBackend
    real = backend_cls.paste
    count = [0]

    def paste(self, *a, **kw):
        real(self, *a, **kw)
        count[0] += 1
        if count[0] == 3:                   # the last round: every tile resumes from host memory
            host.get_shared().state.interrupted = True
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    backend_cls.paste = paste
    try:
        got, st = _run(hook, x, 0)
    finally:
        backend_cls.paste = real
        host.get_shared().state.interrupted = False
    assert sum(st["tiles_parked"].values()) > 0
    assert got.shape == want.shape
    ib, ob = hook.split_tiles(x.shape[2], x.shape[3])
    for i, b in enumerate(ob):            # the forward order of the last round (30 sites: an even number of barriers)
        region = (slice(None), slice(None), slice(b[2], b[3]), slice(b[0], b[1]))
        if i < 3:
            assert_bit_equal(got[region], want[region], f"tile {i}")
        else:
            assert not got[region].any(), f"tile {i} should not have been pasted"
    del got
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == base


def test_short_host_memory_raises_before_any_tile(mods, monkeypatch):
    tv, ve, _ = mods
    hook, x = _case(mods, True, torch.float16)
    runs = []
    real = ve.Executor.run
    monkeypatch.setattr(ve, "host_available_bytes", lambda meminfo="/proc/meminfo": 1 << 20)
    monkeypatch.setattr(ve.Executor, "run", lambda self, st, stop=None: runs.append(1) or real(self, st, stop))
    with pytest.raises(RuntimeError, match="pinned host memory"):
        _run(hook, x, 0)
    assert runs == []
