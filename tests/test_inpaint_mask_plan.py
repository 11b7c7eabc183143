"""Inpainting plan (init_inpaint_mask), host logic on the CPU: which grid tiles and custom regions an inpaint mask reaches,
the compact tile batches and slot table of the sampler loop, the refusals and the progress totals.

The active-tile rule is restated here in numpy (`rule`) and checked against window containment; the device kernel
(td_grid_active_tiles) is pinned against the same restatement by tests/test_gpu_inpaint_mask.py.  Without a device,
engine.active_tiles is replaced by the restatement.
"""
import types

import numpy as np
import pytest
import torch


JUST_BELOW_ONE = 0.99951171875          # the largest fp16 value below 1
GEOMS = [  # W, H, tile, overlap, tile_bs (latent units)
    (128, 96, 48, 16, 4),
    (512, 512, 96, 48, 8),               # cfg2: 100 tiles
    (200, 136, 64, 24, 3),
]


def rule(mask: torch.Tensor, bboxes) -> np.ndarray:
    """A window is active when any mask element in it, over all leading planes, is not exactly 1.0 (NaN is not 1.0)."""
    H, W = mask.shape[-2:]
    m = mask.detach().cpu().float().numpy().reshape(-1, H, W)
    return np.array([bool((m[:, y:y + h, x:x + w] != 1.0).any()) for x, y, w, h in bboxes], dtype=bool)


def _engine():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine      # imported late: the library is built by conftest
    return engine


def _stub_active_tiles(g, mask):
    return rule(mask, [tuple(int(v) for v in r) for r in _engine().grid_bboxes_xywh(g)])


@pytest.fixture(autouse=True)
def _no_device(monkeypatch):
    monkeypatch.setattr(_engine(), "active_tiles", _stub_active_tiles)


def _p(W, H, sampler="Euler a"):
    return types.SimpleNamespace(width=W * 8, height=H * 8, sampler_name=sampler, disable_extra_networks=True, batch_size=1,
                                 steps=20, styles=None, all_prompts=["a photo"], all_negative_prompts=["blurry"])


class _KSampler:
    def __init__(self):
        self.model_wrap_cfg = types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None), image_cfg_scale=None, step=0)


def _delegate(cls, geom, **grid_kw):
    W, H, t, ov, bs = geom
    d = cls(_p(W, H), _KSampler())
    d.init_grid_bbox(t, t, ov, bs, **grid_kw)
    return d


def _bboxes(d):
    return [(b.x, b.y, b.w, b.h) for batch in d.batched_bboxes for b in batch]


def _containing(bboxes, points):
    return np.array([any(x <= px < x + w and y <= py < y + h for py, px in points) for x, y, w, h in bboxes], dtype=bool)


def _methods():
    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion
    return [MultiDiffusion, MixtureOfDiffusers]


# ------------------------------------------------------------------------------------------------ the rule
@pytest.mark.parametrize("geom", GEOMS, ids=[f"{g[0]}x{g[1]}" for g in GEOMS])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
def test_one_element_at_tile_edges_and_corners(geom, dtype):
    """A single element that is not 1 activates exactly the tiles whose window contains it: tile corners, edges on both sides
    of every tile boundary, the canvas corners."""
    W, H = geom[0], geom[1]
    d = _delegate(_methods()[0], geom)
    bbs = _bboxes(d)
    points = {(0, 0), (H - 1, W - 1), (0, W - 1), (H - 1, 0)}
    for x, y, w, h in bbs:
        for py in (y, y + h - 1):
            for px in (x, x + w - 1):
                points.add((py, px))
                for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
                    if 0 <= py + dy < H and 0 <= px + dx < W:
                        points.add((py + dy, px + dx))
    points = sorted(points)
    rng = np.random.default_rng(W * H)
    if len(points) > 64:                                # keep the canvas corners, sample the rest
        points = points[:2] + points[-2:] + [points[i] for i in rng.choice(len(points), 60, replace=False)]
    m = torch.ones((H, W), dtype=dtype)
    for py, px in points:
        for val in (0.0, JUST_BELOW_ONE, float("nan"), 2.0):
            m[py, px] = val
            # bf16 stores 1 - 2^-11 as 1.0 (round to nearest): the rule reads the stored value
            kept = m[py, px].item() == 1.0
            assert kept == (dtype == torch.bfloat16 and val == JUST_BELOW_ONE)
            want = np.zeros(len(bbs), bool) if kept else _containing(bbs, [(py, px)])
            assert np.array_equal(rule(m, bbs), want), (py, px, val)
        m[py, px] = 1.0


@pytest.mark.parametrize("shape", ["hw", "chw", "nchw"])
def test_leading_planes_all_count(shape):
    geom = GEOMS[0]
    W, H = geom[0], geom[1]
    d = _delegate(_methods()[0], geom)
    bbs = _bboxes(d)
    lead = {"hw": (), "chw": (4,), "nchw": (2, 4)}[shape]
    m = torch.ones(lead + (H, W), dtype=torch.float16)
    m.view(-1, H, W)[-1, 40, 70] = 0.5                  # only the last plane differs
    assert np.array_equal(rule(m, bbs), _containing(bbs, [(40, 70)]))
    d.init_inpaint_mask(m)
    assert np.array_equal(d._inpaint.active, _containing(bbs, [(40, 70)]))


@pytest.mark.parametrize("fill, want", [(1.0, False), (0.0, True), (float("nan"), True), (JUST_BELOW_ONE, True)])
def test_uniform_masks(fill, want):
    geom = GEOMS[1]
    d = _delegate(_methods()[0], geom)
    d.init_inpaint_mask(torch.full((1, 4, geom[1], geom[0]), fill, dtype=torch.float16))
    assert d._inpaint.active.tolist() == [want] * d.num_tiles


def test_cfg2_centre_square_count():
    """cfg2's geometry (latent 512^2, tile 96, overlap 48): a mask touching the 128^2 latent square in the middle."""
    d = _delegate(_methods()[0], GEOMS[1])
    m = torch.ones((512, 512), dtype=torch.float16)
    m[192:320, 192:320] = 0
    d.init_inpaint_mask(m)
    n = int(d._inpaint.active.sum())
    print(f"cfg2: {n} of {d.num_tiles} tiles active, {len(d._inpaint.batched_bboxes)} of {d.num_batches} UNet batches")
    assert n == 16 and d.num_tiles == 100


# ------------------------------------------------------------------------------------------------ compact batches, slots
@pytest.mark.parametrize("geom", GEOMS, ids=[f"{g[0]}x{g[1]}" for g in GEOMS])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_compact_batches_and_slot_table(geom, seed):
    W, H = geom[0], geom[1]
    for cls in _methods():
        d = _delegate(cls, geom)
        bbs = _bboxes(d)
        rng = np.random.default_rng(seed)
        m = torch.ones((H, W), dtype=torch.float32)
        for _ in range(int(rng.integers(1, 6))):
            m[int(rng.integers(0, H)), int(rng.integers(0, W))] = 0
        d.init_inpaint_mask(m)
        ip = d._inpaint
        tiles = [t for t in range(d.num_tiles) if ip.active[t]]
        assert ip.tiles == tiles
        assert ip.slot_host.dtype == np.int32 and ip.slot_host.tolist() == [tiles.index(t) if ip.active[t] else -1 for t in range(d.num_tiles)]
        assert torch.equal(ip.slot_dev.cpu(), torch.from_numpy(ip.slot_host))
        flat = [(b.x, b.y, b.w, b.h) for batch in ip.batched_bboxes for b in batch]
        assert flat == [bbs[t] for t in tiles]
        assert [len(b) for b in ip.batched_bboxes] == [min(d.tile_bs, len(tiles) - i) for i in range(0, len(tiles), d.tile_bs)]
        assert ip.origins_dev.tolist() == [v for t in tiles for v in bbs[t][:2]]
        assert list(ip.origins_host)[:2 * len(tiles)] == ip.origins_dev.tolist()
        # the full plan stays what init_grid_bbox made (noise inversion and the weight canvas use it)
        assert _bboxes(d) == bbs
        assert d._active_plan() is ip
        d._full_plan_pass = True                       # noise inversion runs the full plan
        assert d._active_plan() is None


def test_slot_table_helper():
    a = np.array([False, True, True, False, True])
    assert _engine().slot_table(a).tolist() == [-1, 0, 1, -1, 2]
    assert _engine().slot_table(np.zeros(3, bool)).tolist() == [-1, -1, -1]


# ------------------------------------------------------------------------------------------------ regions
def _rows():
    from multidiffusion_upscaler_for_automatic1111_b200.tile_utils.utils import BlendMode
    bg, fg = BlendMode.BACKGROUND.value, BlendMode.FOREGROUND.value
    return {0: (True, 0.0, 0.0, 0.25, 0.25, "top left", "", bg, 0.2, -1),
            1: (True, 0.6, 0.6, 0.4, 0.4, "bottom right", "", fg, 0.3, 5),
            2: (True, 0.3, 0.0, 0.3, 0.5, "top", "", bg, 0.2, -1)}


@pytest.mark.parametrize("draw_background", [True, False])
def test_regions_skipped_and_kept(draw_background):
    geom = GEOMS[0]
    W, H = geom[0], geom[1]
    for cls in _methods():
        d = _delegate(cls, geom)
        d.init_custom_bbox(_rows(), draw_background, False)
        rects = [(b.x, b.y, b.w, b.h) for b in d.custom_bboxes]
        m = torch.ones((H, W), dtype=torch.bfloat16)
        py, px = H - 2, W - 2                          # inside region 1 only
        m[py, px] = 0
        w_before = d.weights.clone()
        d.init_inpaint_mask(m)
        want = rule(m, rects)
        assert d._inpaint.regions == want.tolist() == [False, True, False]
        assert torch.equal(d.weights, w_before)        # the weight canvas (BACKGROUND +1 / gaussians included) stays the full plan's
        assert [d._region_skipped(i) for i in range(3)] == [True, False, True]
        if not draw_background:
            assert d._inpaint.batched_bboxes == [] and d._inpaint.active.shape == (0,)
        # the region pass drops the skipped regions (and with them their composite terms)
        calls = []
        done = d._custom_region_pass(torch.zeros((1, 4, H, W)), lambda x, i, b: calls.append(i) or x, poll_interrupt=False)
        assert calls == [1] and [i for i, _, _ in done] == [1]


# ------------------------------------------------------------------------------------------------ refusals
def _assert_refused(d, exc, mask):
    before = dict(d.__dict__)
    with pytest.raises(exc):
        d.init_inpaint_mask(mask)
    assert d.__dict__.keys() == before.keys() and all(d.__dict__[k] is before[k] for k in before), "refusal changed state"


def test_refusals_leave_state_unchanged():
    from multidiffusion_upscaler_for_automatic1111_b200 import parallel
    geom = GEOMS[0]
    W, H = geom[0], geom[1]
    ok = torch.ones((H, W), dtype=torch.float16)
    for cls in _methods():
        d = _delegate(cls, geom)
        for bad in (torch.ones((H, W + 1)), torch.ones((H + 8, W)), torch.ones((W, H)), torch.ones((2, 1, 4, H, W)),
                    torch.ones((W * H,)), torch.ones((H, W), dtype=torch.float64), torch.ones((H, W), dtype=torch.int32), None):
            _assert_refused(d, ValueError, bad)
        _assert_refused(_delegate(cls, geom, wrap_x=True), NotImplementedError, ok)
        _assert_refused(_delegate(cls, geom, wrap_y=True), NotImplementedError, ok)
        sh = _delegate(cls, geom)
        sh._shard = parallel.TileShard(sh.num_tiles, 0, 2)       # what init_tile_shard leaves
        _assert_refused(sh, NotImplementedError, ok)
        # the other order: the shard after the mask
        d.init_inpaint_mask(ok)
        before = dict(d.__dict__)
        with pytest.raises(NotImplementedError):
            d.init_tile_shard(None, mode="replicate")
        assert d.__dict__.keys() == before.keys() and all(d.__dict__[k] is before[k] for k in before)


def test_spot_and_demofusion_refuse():
    from multidiffusion_upscaler_for_automatic1111_b200 import DemoFusion, SpotDiffusion
    geom = GEOMS[0]
    W, H = geom[0], geom[1]
    s = SpotDiffusion(_p(W, H), _KSampler())
    s.init_grid_bbox(48, 48, 16, 4)
    _assert_refused(s, NotImplementedError, torch.ones((H, W), dtype=torch.float16))
    df = DemoFusion.__new__(DemoFusion)          # the refusal needs no state at all
    df.__dict__["marker"] = 1
    _assert_refused(df, NotImplementedError, torch.ones((H, W), dtype=torch.float16))


# ------------------------------------------------------------------------------------------------ progress totals
@pytest.mark.parametrize("draw_background", [True, False])
def test_progress_totals(draw_background):
    geom = GEOMS[1]
    W, H = geom[0], geom[1]
    for cls in _methods():
        d = _delegate(cls, geom)
        d.init_custom_bbox(_rows(), draw_background, False)
        m = torch.ones((H, W))
        m[300:320, 300:330] = 0.25                       # inside region 1 (bottom right) only
        d.init_inpaint_mask(m)
        d.init_done()
        ip = d._inpaint
        want = (len(ip.batched_bboxes) if draw_background else 0) + sum(ip.regions)
        assert d.total_bboxes == want and sum(ip.regions) == 1
        assert len(ip.batched_bboxes) == -(-int(ip.active.sum()) // d.tile_bs) < d.num_batches

        # a mask that keeps everything: nothing to denoise, and init_done accepts it
        k = _delegate(cls, geom)
        k.init_custom_bbox(_rows(), draw_background, False)
        k.init_inpaint_mask(torch.ones((1, 4, H, W), dtype=torch.float16))
        k.init_done()
        assert k.total_bboxes == 0 and k._inpaint.batched_bboxes == [] and not any(k._inpaint.regions)


def test_without_mask_totals_unchanged():
    geom = GEOMS[1]
    for cls in _methods():
        d = _delegate(cls, geom)
        d.init_done()
        assert d._inpaint is None and d._active_plan() is None and d.total_bboxes == d.num_batches
