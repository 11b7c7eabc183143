"""Batched tensor-core VAE pass on the host: how many images go through the tiles together (VAEHook._images_per_pass),
the per-pass shape walk, and the per-image merge of GroupNorm statistics (no GPU needed)."""
import os

import pytest
import torch

from oracle import ldm_vae


@pytest.fixture(scope="module")
def mods():
    from multidiffusion_upscaler_for_automatic1111_b200 import tilevae, vae_engine
    return tilevae, vae_engine


@pytest.fixture(scope="module")
def dec_program(mods):
    return mods[1].compile_program(ldm_vae.Decoder(), True)


def test_pick_takes_the_largest_count_that_fits(mods):
    tv, _ = mods
    assert tv.pick_images_per_pass(4, lambda k: True) == 4
    assert tv.pick_images_per_pass(4, lambda k: k <= 3) == 3
    assert tv.pick_images_per_pass(8, lambda k: k <= 2) == 2
    assert tv.pick_images_per_pass(4, lambda k: False) == 1
    asked = []
    assert tv.pick_images_per_pass(1, lambda k: asked.append(k) or True) == 1
    assert asked == []          # one image: nothing to decide


def test_footprint_of_a_batched_pass(mods, dec_program):
    _, ve = mods
    one = ve.tile_footprint(dec_program, "wgmma", torch.float16, 40, 52)
    # existing callers: the tensor-core arm ignores `batch` unless the pass's image count is given
    assert ve.tile_footprint(dec_program, "wgmma", torch.float16, 40, 52, 3) == one
    assert ve.tile_footprint(dec_program, "wgmma", torch.float16, 40, 52, 3, images=1) == one
    three = ve.tile_footprint(dec_program, "wgmma", torch.float16, 40, 52, 3, images=3)
    assert three.act == [3 * a for a in one.act] and three.skip == [3 * s for s in one.skip] and three.alias == one.alias
    assert three.working == 3 * one.working          # the peak is a convolution at full resolution here
    # the module backend still takes the batch as it did
    assert ve.tile_footprint(dec_program, "modules", torch.float32, 40, 52, 3, images=1) == \
        ve.tile_footprint(dec_program, "modules", torch.float32, 40, 52, 3)


class _Backend:
    name = "wgmma"
    dtype = torch.float16


def _hook(tv, fast=False, color_fix=False):
    net = ldm_vae.Decoder()
    hook = tv.VAEHook(net, 8, True, fast_decoder=fast, fast_encoder=fast, color_fix=color_fix)
    return hook


@pytest.mark.parametrize("fast", [False, True], ids=["slow", "fast"])
def test_images_per_pass_follows_memory(mods, dec_program, monkeypatch, fast):
    tv, ve = mods
    hook = _hook(tv, fast)
    z = torch.empty((4, 4, 40, 52))
    ib, _ = hook.split_tiles(40, 52)
    monkeypatch.setattr(tv.VAEHook, "_free_bytes", staticmethod(lambda dev: 1 << 40))
    assert hook._images_per_pass(dec_program, _Backend(), z, ib) == 4
    # room for the working set of two images and every tile of two images resident, not three
    fps = {k: [ve.tile_footprint(dec_program, "wgmma", torch.float16, b[3] - b[2], b[1] - b[0], k, images=k) for b in ib]
           for k in (2, 3)}
    need = {k: max(f.working for f in fps[k]) + 2 * max(f.held(s) for f in fps[k] for s in range(dec_program.num_sites)) +
            max(sum(max(f.resident(s), f.resident(max(s - 1, 0))) for f in fps[k]) for s in range(dec_program.num_sites))
            for k in (2, 3)}
    free = need[2] if not fast else max(f.working for f in fps[2])
    monkeypatch.setattr(tv.VAEHook, "_free_bytes", staticmethod(lambda dev: free))
    assert hook._images_per_pass(dec_program, _Backend(), z, ib) == 2
    monkeypatch.setattr(tv.VAEHook, "_free_bytes", staticmethod(lambda dev: 1 << 20))
    assert hook._images_per_pass(dec_program, _Backend(), z, ib) == 1
    # a forced count is clamped to the batch
    monkeypatch.setattr(tv.VAEHook, "_free_bytes", staticmethod(lambda dev: 1 << 40))
    for forced, want in ((1, 1), (3, 3), (9, 4), (0, 1)):
        hook.images_per_pass = forced
        assert hook._images_per_pass(dec_program, _Backend(), z, ib) == want


def test_a_budget_that_would_park_keeps_one_image_per_pass(mods, dec_program, monkeypatch):
    """Slow mode: parking copies through host memory, so a budget the batched pass would have to park under keeps one
    image per pass even though the working set fits."""
    tv, _ = mods
    hook = _hook(tv)
    ib, _ = hook.split_tiles(40, 52)
    monkeypatch.setattr(tv.VAEHook, "_free_bytes", staticmethod(lambda dev: 1 << 40))
    hook.max_resident_bytes = 0
    assert hook._images_per_pass(dec_program, _Backend(), torch.empty((3, 4, 40, 52)), ib) == 1
    # fast mode without color fix has no barrier: nothing is ever parked
    fast = _hook(tv, fast=True)
    fast.max_resident_bytes = 0
    assert fast._images_per_pass(dec_program, _Backend(), torch.empty((3, 4, 40, 52)), ib) == 3
    # with color fix (an encoder's) the sites from the first down-sampling on stay barriers; a decoder has none of those
    _, end = mods[1].estimated_ops(dec_program, True)
    assert end == max(i for i, op in enumerate(dec_program.ops) if isinstance(op, mods[1].Norm)) + 1


def _stats(seed, tiles, images):
    g = torch.Generator().manual_seed(seed)
    var = [torch.rand(images * 32, generator=g) * 10 ** torch.randint(-3, 3, (1,), generator=g).item() for _ in range(tiles)]
    mean = [torch.randn(images * 32, generator=g) * 100 for _ in range(tiles)]
    px = [int(v) for v in torch.randint(1, 5000, (tiles,), generator=g)]
    return var, mean, px


def _param(tv, var, mean, px, group=None, sharded=False):
    p = tv.GroupNormParam(group, sharded)
    for v, m, n in zip(var, mean, px):
        p.add(v, m, n)
    return p


@pytest.mark.parametrize("images", [2, 3, 8])
def test_per_image_merge_is_the_one_image_merge(mods, images):
    tv, _ = mods
    var, mean, px = _stats(images, 7, images)
    got_mean, got_var = _param(tv, var, mean, px).summary(32 * images, None, images)
    for j in range(images):
        sl = slice(32 * j, 32 * (j + 1))
        want_mean, want_var = _param(tv, [v[sl].clone() for v in var], [m[sl].clone() for m in mean], px).summary(32)
        assert torch.equal(got_mean[sl], want_mean) and torch.equal(got_var[sl], want_var), f"image {j}"
    assert tv.GroupNormParam().summary(64, None, 2) is None


def test_per_image_merge_under_the_tile_shard(mods, tmp_path):
    """One all-reduce per image, each packed as a one-image pass packs it (one rank of a gloo group on the CPU)."""
    import torch.distributed as dist
    tv, _ = mods
    dist.init_process_group("gloo", init_method=f"file://{os.path.join(tmp_path, 'store')}", world_size=1, rank=0)
    try:
        var, mean, px = _stats(5, 4, 3)
        got_mean, got_var = _param(tv, var, mean, px, sharded=True).summary(96, None, 3)
        for j in range(3):
            sl = slice(32 * j, 32 * (j + 1))
            want_mean, want_var = _param(tv, [v[sl].clone() for v in var], [m[sl].clone() for m in mean], px, sharded=True).summary(32)
            assert torch.equal(got_mean[sl], want_mean) and torch.equal(got_var[sl], want_var)
        # a rank without tiles still joins every image's all-reduce
        empty_mean, empty_var = tv.GroupNormParam(None, True).summary(96, torch.device("cpu"), 3)
        assert empty_mean.shape == (96,) and empty_var.shape == (96,)
    finally:
        dist.destroy_process_group()
