"""Tiled-VAE residency plan on the host: the shape walk of the compiled program (bytes a tile holds at each GroupNorm
site, in the backends' layouts) and the choice of the tiles that wait in host memory at each barrier."""
import pytest
import torch

from oracle import ldm_vae, vae


@pytest.fixture(scope="module")
def ve():
    from multidiffusion_upscaler_for_automatic1111_b200 import vae_engine
    return vae_engine


@pytest.fixture(scope="module")
def programs(ve):
    return {dec: ve.compile_program((ldm_vae.Decoder if dec else ldm_vae.Encoder)(), dec) for dec in (True, False)}


def _tiles(is_dec, size, tile):
    ib, _ = vae.split_tiles(size, size, tile, 11 if is_dec else 32, is_dec)
    return [(b[3] - b[2], b[1] - b[0]) for b in ib]


def _worst_site_total(ve, prog, backend, dtype, tiles):
    fps = [ve.tile_footprint(prog, backend, dtype, h, w) for h, w in tiles]
    return max(sum(f.held(s) for f in fps) for s in range(prog.num_sites))


# decoder z edge / encoder image edge, tile, tiles, GB held at the worst site (fp16 wgmma, fp32 modules)
SD_CASES = [(True, 1024, 96, 121, 76.1, 152.1), (True, 1024, 256, 16, 58.4, 116.8), (True, 1536, 96, 256, 171.1, 342.3),
            (False, 8192, 1536, 36, 37.1, 74.2), (False, 12288, 1536, 64, 83.0, 166.1)]


@pytest.mark.parametrize("is_dec,size,tile,n,gb16,gb32", SD_CASES)
def test_shape_walk_peaks_of_the_sd_layout(ve, programs, is_dec, size, tile, n, gb16, gb32):
    tiles = _tiles(is_dec, size, tile)
    assert len(tiles) == n
    prog = programs[is_dec]
    assert _worst_site_total(ve, prog, "wgmma", torch.float16, tiles) / 1e9 == pytest.approx(gb16, abs=0.05)
    assert _worst_site_total(ve, prog, "modules", torch.float32, tiles) / 1e9 == pytest.approx(gb32, abs=0.05)


def test_shape_walk_layouts(ve, programs):
    dec = programs[True]
    # cfg4's widest site: the first level-0 block's norm1, a 256-channel input beside its 128-channel nin_shortcut
    fp = ve.tile_footprint(dec, "wgmma", torch.float16, 118, 118)
    widest = max(range(dec.num_sites), key=fp.held)
    assert fp.act[widest] == 944 * 944 * 256 * 2 and fp.skip[widest] == 944 * 944 * 128 * 2
    # the mid-block attention's norm: an identity shortcut is the activation itself, counted once
    attn = [op.site for op, nxt in zip(dec.ops, dec.ops[1:]) if isinstance(op, ve.Norm) and isinstance(nxt, ve.Attention)][0]
    assert fp.skip[attn] == 0 and fp.act[attn] == 118 * 118 * 512 * 2 and fp.alias[attn]
    # once that norm is applied, the normalised activation sits beside the shortcut
    assert fp.resident(attn) == 2 * fp.held(attn) and fp.resident(widest) == fp.held(widest)
    # the working set includes the four-GEMM attention's [T, round_up(T, 8)] score matrix
    T = 118 * 118
    assert fp.working >= T * ve.ops.round_up(T, 8) * 2
    # NCHW, batch 2, exact channels, fp32
    fm = ve.tile_footprint(dec, "modules", torch.float32, 118, 118, batch=2)
    assert fm.held(widest) == 2 * 2 * fp.held(widest)
    # the encoder's conv_in input is padded from 3 to 64 channels on the tensor cores
    enc = programs[False]
    fe = ve.tile_footprint(enc, "wgmma", torch.float16, 64, 64)
    assert fe.working >= 64 * 64 * 64 * 2 + 64 * 64 * 128 * 2


def _orders(n, rounds):
    return [list(range(n)) if r % 2 == 0 else list(range(n - 1, -1, -1)) for r in range(rounds)]


def _sd_held(ve, programs, is_dec, size, tile):
    prog = programs[is_dec]
    tiles = _tiles(is_dec, size, tile)
    fps = [ve.tile_footprint(prog, "wgmma", torch.float16, h, w) for h, w in tiles]
    return [[f.resident(s) for f in fps] for s in range(prog.num_sites)]


@pytest.mark.parametrize("frac", [0.0, 0.1, 0.33, 0.5, 0.9])
def test_plan_fits_the_budget_and_keeps_a_suffix(ve, programs, frac):
    held = _sd_held(ve, programs, True, 1024, 96)
    orders = _orders(len(held[0]), len(held))
    budget = int(frac * max(sum(h) for h in held))
    parked = ve.plan_residency(orders, held, budget)
    prev = {}
    for r, order in enumerate(orders):
        p = parked[r]
        # Belady under the zig-zag: the parked tiles are a prefix of the round's order, the resident ones its suffix
        assert p == order[:len(p)]
        resident = order[len(p):]
        assert sum(held[r][i] for i in resident) <= budget
        # and at every point of the round: previous residents not yet visited + new residents already visited
        for k in range(len(order) + 1):
            now = sum(prev.get(i, 0) for i in order[k:]) + sum(held[r][i] for i in order[:k] if i in set(resident))
            assert now <= budget
        prev = {i: held[r][i] for i in resident}
    if frac < 0.5:
        assert sum(len(p) for p in parked) > 0


def test_plan_keeps_the_most_that_fits(ve):
    """Equal tiles: exactly floor(budget / tile) stay resident at every barrier."""
    held = [[10] * 7 for _ in range(4)]
    parked = ve.plan_residency(_orders(7, 4), held, 35)
    assert [len(p) for p in parked] == [4, 4, 4, 4]
    assert parked[0] == [0, 1, 2, 3] and parked[1] == [6, 5, 4, 3]


@pytest.mark.parametrize("is_dec,size,tile", [(True, 1024, 96), (False, 8192, 1536)])
def test_plan_budget_at_least_total_parks_nothing(ve, programs, is_dec, size, tile):
    held = _sd_held(ve, programs, is_dec, size, tile)
    orders = _orders(len(held[0]), len(held))
    total = max(sum(h) for h in held)
    assert not any(ve.plan_residency(orders, held, total))
    assert not any(ve.plan_residency(orders, held, 10 * total))
    assert all(len(p) == len(held[0]) for p in ve.plan_residency(orders, held, 0))


def test_uniform_budget_at_total_parks_nothing(ve):
    held = [[5] * 9, [7] * 9, [3] * 9]
    assert not any(ve.plan_residency(_orders(9, 3), held, 63))


def test_host_memory_check(ve, tmp_path):
    f = tmp_path / "meminfo"
    f.write_text("MemTotal:       65536000 kB\nMemFree:        1000 kB\nMemAvailable:   2048 kB\n")
    none = str(tmp_path / "no-cgroup")
    assert ve.host_available_bytes(str(f), none) == 2048 * 1024
    assert ve.host_available_bytes(str(tmp_path / "missing"), none) is None
    cg = tmp_path / "cg"
    cg.mkdir()
    (cg / "memory.max").write_text("3145728\n")
    (cg / "memory.current").write_text("2097152\n")
    assert ve.host_available_bytes(str(tmp_path / "missing"), str(cg)) == 1 << 20      # a container's cap counts
    assert ve.host_available_bytes(str(f), str(cg)) == 1 << 20
    (cg / "memory.max").write_text("max\n")
    assert ve.host_available_bytes(str(f), str(cg)) == 2048 * 1024
    ve.require_host_memory(2048 * 1024, 2048 * 1024)
    with pytest.raises(RuntimeError, match=r"pinned host memory"):
        ve.require_host_memory(10 * 2 ** 30, 2048 * 1024)
