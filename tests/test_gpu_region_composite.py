"""td_region_composite / td_region_composite_rows (csrc/td_region.cu, engine.region_composite / region_composite_rows) at
every canvas x region-output dtype pair, every size class of the grid-stride loop, the region limits, the geometry and value
edges, and every refusal -- against helpers.region_composite_reference (the reference's tensor expressions,
multidiffusion.py:187-216 / mixtureofdiffusers.py:145-175, run by torch on the CPU: IEEE fp32, no FMA).

Every comparison is bit-exact.  Where a NaN is expected the NaN positions are compared and then the bits of every other
element (CPU and GPU NaN payloads differ; assert_bit_equal's signed-zero opt-out would hide the signed zeros too).

The CPU test at the top shows that the hand-placed value-edge inputs tell the real composite apart from five plausible
wrong ones, so that the GPU tests passing on them means something."""
import numpy as np
import pytest
import torch

from helpers import DTYPES, assert_bit_equal, region_composite_reference
from oracle import region, synth, tiling
from oracle.make_golden import REGION_CASES, REGION_GRID

gpu = pytest.mark.gpu

GRID_CAP = 148 * 16 * 256           # elements one pass of the launch's capped grid covers
SPLITS = [("f16", "f32"), ("bf16", "f32"), ("bf16", "f16")]   # (canvas, output) pairs where rounding the output first shows


def _same(got, want, what):
    """Bit equality, with NaN compared by position only."""
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype}{tuple(got.shape)} vs {want.dtype}{tuple(want.shape)}"
    gn, wn = got.isnan(), want.isnan()
    assert torch.equal(gn, wn), f"{what}: NaN positions differ at {int((gn ^ wn).sum())} elements"
    assert_bit_equal(got.masked_fill(gn, 0.0), want.masked_fill(wn, 0.0), what)


def _differs(a, b) -> bool:
    an, bn = a.isnan(), b.isnan()
    return not torch.equal(an, bn) or not np.array_equal(a.masked_fill(an, 0.0).numpy().view(np.uint32),
                                                         b.masked_fill(bn, 0.0).numpy().view(np.uint32))


def _cuda(regions):
    return [(x, y, w, h, m, o.cuda(), None if a is None else a.cuda()) for (x, y, w, h, m, o, a) in regions]


def _run(xb, weights, regions):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    return engine.region_composite(xb.cuda(), None if weights is None else weights.cuda(), _cuda(regions)).cpu()


def _run_rows(xb, weights, regions, windows):
    """The rows entry over each window into its own NaN-sentinel canvas: rows outside the window must stay NaN.  Returns the
    union of the windows' rows (NaN where no window reached)."""
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N, C, H, W = xb.shape
    xd, wd, rd = xb.cuda(), None if weights is None else weights.cuda(), _cuda(regions)
    union = torch.full((N, C, H, W), float("nan"))
    for lo, hi in windows:
        got = engine.region_composite_rows(xd, wd, rd, lo, hi, torch.full((N, C, H, W), float("nan"), device="cuda")).cpu()
        outside = torch.cat([got[:, :, :lo], got[:, :, hi:]], dim=2)
        assert bool(outside.isnan().all()), f"rows window [{lo},{hi}) wrote outside itself"
        union[:, :, lo:hi] = got[:, :, lo:hi]
    return union


def _check_both_entries(xb, weights, regions, what, windows=None):
    want = region_composite_reference(xb, weights, regions)
    _same(_run(xb, weights, regions), want, what)
    H = xb.shape[2]
    if windows is None:
        a = min(3, H - 1)
        windows = [(0, 0), (0, a), (a, H - 1), (H - 1, H)]
    union = _run_rows(xb, weights, regions, windows)
    covered = torch.zeros(H, dtype=torch.bool)
    for lo, hi in windows:
        covered[lo:hi] = True
    _same(union[:, :, covered], want[:, :, covered], what + " (rows entry)")
    return want


# ------------------------------------------------------------------------------------------------ hand-placed value edges
def _t(rows, dt=torch.float32):
    return torch.tensor(rows, dtype=torch.float32).to(dt)


def value_edge_cases(dn):
    """[(name, x_buffer, weights, regions)] of canvas dtype `dn`, fp32 region outputs unless stated; [1, 1, 4, 8] canvases."""
    T = DTYPES[dn]
    nan, inf = float("nan"), float("inf")
    cases = []
    # MultiDiffusion: BACKGROUND adds and the divide-where->1 normalisation, FOREGROUND over it
    xb = _t([[-0.0, 0.0, -0.0, 0.0, 65504.0, -60000.0, 0.1, 3.0],            # signed zeros, fp16 overflow, weight 2 and 0.5
             [-0.0, -0.0, 0.0, -0.0, 2.5, -0.0, 1.0, 7.0],                    # FOREGROUND over +-0 with mask 0 and 1
             [0.75, 1.5, -0.5, 2.0, 0.0, 1.0, -3.0, 0.25],                    # two overlapping FOREGROUNDs (fb rounding)
             [0.1, 0.7, -1.3, 2.9, -0.3, 5.5, 0.45, -7.1]], T).view(1, 1, 4, 8)
    weights = _t([[1.0, 1.0, 1.0, 1.0, 1.0, 2.0, 3.0, 0.5],
                  [1.0, 1.0, 1.0, 1.0, 0.0, 1.0, 1.0, 0.5],
                  [0.0, 2.0, 1.0, 0.5, 4.0, 1.0, 1.0, 3.0],
                  [1.0, 0.5, 3.0, 0.0, 2.0, 1.0, 4.0, 1.0]])
    bg0 = _t([[-0.0, -0.0, 0.0, 0.0, 16.0, 70000.0, 1.0 / 3.0, 1.0]]).view(1, 1, 1, 8)
    fg1 = _t([[0.0, 5.0, -0.0, -0.0, 1.25, nan, inf, 3.0]]).view(1, 1, 1, 8)
    m1 = _t([[0.0, 0.0, 1.0, 1.0, 0.5, 0.0, 0.25, 0.3]])
    fg2a = _t([[1.0, 1.0, 1.0, 1.0, -2.0, 0.5, 3.0, 1.0]]).view(1, 1, 1, 8)
    fg2b = _t([[2.0 ** -11, 2.0 ** -9, 3 * 2.0 ** -12, 2.0 ** -8 + 2.0 ** -12, -(2.0 ** -10), 2.0 ** -12, 2.0 ** -8, 0.1]]).view(1, 1, 1, 8)
    m2a, m2b = _t([[0.2, 0.4, 0.6, 1.0, 0.0, 0.3, 0.9, 0.7]]), _t([[0.5, 0.1, 0.25, 1.0, 0.0, 0.45, 0.35, 0.15]])
    fg3 = _t([[1.0 / 3.0, -0.7, 2.2, 0.123, 9.75, -4.4, 0.9, 1.7]]).view(1, 1, 1, 8)
    m3 = _t([[0.1, 0.2, 0.3, 0.35, 0.45, 0.55, 0.65, 0.9]])
    bg3 = _t([[0.3, 0.6, -0.9, 1.2, 0.0, 2.2, -0.7, 0.05]]).view(1, 1, 1, 8)
    cases.append(("md", xb, weights, [(0, 0, 8, 1, 0, bg0, None), (0, 3, 8, 1, 0, bg3, None), (0, 1, 8, 1, 1, fg1, m1),
                                      (0, 2, 8, 1, 1, fg2a, m2a), (0, 2, 8, 1, 1, fg2b, m2b), (0, 3, 8, 1, 1, fg3, m3)]))
    # Mixture of Diffusers: BACKGROUND times its fp32 weights ([1,1,h,w] and [h,w] forms), subnormal products, no normalisation
    xb = _t([[0.0, -0.0, 1.0, -1.0, 0.5, 2.0 ** -130, -0.0, 100.0],
             [-0.0, 0.0, 0.25, 0.0, -0.0, 1.5, 3.0, -2.0]], T).view(1, 1, 2, 8)
    sub = _t([[1e-30, -1e-30, 2.0 ** -70, 3.0, 1.0 / 3.0, 2.0 ** -100, -0.0, 65504.0]]).view(1, 1, 1, 8)
    aux4 = _t([[1e-10, 1e-10, 2.0 ** -70, 2.0 ** -140, 0.3, 2.0 ** -30, 0.7, 1.5]]).view(1, 1, 1, 8)
    bgb = _t([[-0.0, 0.0, 1.0 / 7.0, 0.0, -0.0, nan, 2.0, -inf]]).view(1, 1, 1, 8)
    aux2 = _t([[0.0, 1.0, 0.6, 0.0, 1.0, 1.0, 0.4, 0.5]])
    fgm = _t([[-0.0, 0.0, 0.75, 2.0, 0.0, -1.0, 0.3, 1.0]]).view(1, 1, 1, 8)
    mm = _t([[0.0, 0.0, 0.5, 1.0, 0.0, 0.0, 0.8, 0.0]])
    cases.append(("mod", xb, None, [(0, 0, 8, 1, 0, sub, aux4), (0, 1, 8, 1, 0, bgb, aux2), (0, 1, 8, 1, 1, fgm, mm),
                                    (0, 0, 8, 1, 1, fgm.clone(), mm.clone())]))
    # an output of another dtype than the canvas: a bf16 output above 65504 stays finite in the fp32 add
    xb = _t([[-60000.0, -1.0, 0.0, 65504.0]], T).view(1, 1, 1, 4)
    bf = _t([[70144.0, 1.0 + 2.0 ** -7, -0.0, -70144.0]], torch.bfloat16).view(1, 1, 1, 4)
    cases.append(("bf16_output", xb, None, [(0, 0, 4, 1, 0, bf, None)]))
    return cases


def _restated(x_buffer, weights, regions, mutation=None):
    """region_composite_reference restated with one deliberate defect switched on (`mutation`):
    cast_outputs  region output rounded to the canvas dtype before its add (the defect this file pins)
    fma           the overlay's product and sum contracted into one rounding
    divide_gt0    divide wherever the weight is above 0 (the reference: above 1; dividing by exactly 1 is the identity, so
                  a weight in (0, 1) is what a wrong threshold shows on)
    fb_f32        FOREGROUND outputs summed in fp32 instead of rounding through the canvas dtype
    fm_gate       the overlay applied where the feather mask is above 0 instead of where a FOREGROUND covers the pixel"""
    N, C, H, W = x_buffer.shape
    buf = x_buffer.clone()
    fb = fm = fc = None
    for (x, y, w, h, mode, r_out, aux) in regions:
        if mutation == "cast_outputs":
            r_out = r_out.to(buf.dtype)
        sl = (slice(None), slice(None), slice(y, y + h), slice(x, x + w))
        if mode == 0:
            buf[sl] += r_out if aux is None else r_out * aux
        else:
            if fb is None:
                fb = torch.zeros(buf.shape, dtype=torch.float32 if mutation == "fb_f32" else buf.dtype)
                fm, fc = torch.zeros((1, 1, H, W)), torch.zeros((1, 1, H, W))
            fb[sl] += r_out
            fm[sl] += aux
            fc[sl] += 1
    res = buf
    if weights is not None:
        wv = weights.view(1, 1, H, W)
        res = torch.where(wv > 0 if mutation == "divide_gt0" else wv > 1, buf / wv, buf)
    if fb is not None:
        fb = torch.where(fc > 1, fb / fc, fb)
        fm = torch.where(fc > 1, fm / fc, fm)
        if mutation == "fma":     # one rounding: the fp32 x fp32 product is exact in float64
            over = (res.double() * (1 - fm).double() + (fb * fm).double()).float()
        else:
            over = res * (1 - fm) + fb * fm
        res = torch.where(fm > 0 if mutation == "fm_gate" else fc > 0, over, res)
    return res.float()


MUTATIONS = ["cast_outputs", "fma", "divide_gt0", "fb_f32", "fm_gate"]


def test_value_edge_inputs_tell_wrong_composites_apart():
    """CPU: the restatement without a defect is the reference bit for bit; each defect changes at least one element of
    the hand-placed cases."""
    shown = {m: [] for m in MUTATIONS}
    for dn in DTYPES:
        for name, xb, weights, regions in value_edge_cases(dn):
            want = region_composite_reference(xb, weights, regions)
            _same(_restated(xb, weights, regions), want, f"restatement {dn} {name}")
            for m in MUTATIONS:
                if _differs(_restated(xb, weights, regions, m), want):
                    shown[m].append(f"{dn}/{name}")
    assert all(shown.values()), f"mutations no hand-placed case tells apart: {[m for m, v in shown.items() if not v]}"


@gpu
@pytest.mark.parametrize("dn", list(DTYPES))
def test_value_edges(dn):
    for name, xb, weights, regions in value_edge_cases(dn):
        H = xb.shape[2]
        _check_both_entries(xb, weights, regions, f"{dn} {name}", windows=[(r, r + 1) for r in range(H)])


# ------------------------------------------------------------------------------------------------ dtype matrix
LAYOUTS = {   # name: (MultiDiffusion weights?, [(x, y, w, h, mode, aux form)]); aux form: None | "4d" | "2d" | "mask"
    "md_background": (True, [(3, 2, 20, 17, 0, None), (0, 0, 56, 40, 0, None), (8, 30, 9, 7, 0, None), (40, 20, 16, 20, 0, None)]),
    "mod_background_4d": (False, [(3, 2, 20, 17, 0, "4d"), (0, 0, 56, 40, 0, "4d"), (8, 30, 9, 7, 0, "4d")]),
    "mod_background_2d": (False, [(3, 2, 20, 17, 0, "2d"), (10, 8, 30, 25, 0, "2d"), (40, 20, 16, 20, 0, "2d")]),
    "foreground_only": (False, [(10, 8, 30, 25, 1, "mask"), (25, 5, 24, 30, 1, "mask"), (40, 20, 16, 20, 1, "mask")]),
    "mixed": (True, [(3, 2, 20, 17, 0, None), (10, 8, 30, 25, 1, "mask"), (0, 0, 56, 40, 0, "4d"), (25, 5, 24, 30, 1, "mask"),
                     (40, 20, 16, 20, 1, "mask"), (8, 30, 9, 7, 0, "2d")]),
}


def _random_case(seed, N, C, H, W, canvas_dn, out_dn, rects, with_weights):
    g = torch.Generator().manual_seed(seed)
    xb = (torch.randn((N, C, H, W), generator=g) * 2).to(DTYPES[canvas_dn])
    weights = torch.randint(0, 9, (H, W), generator=g).float() * 0.5 if with_weights else None     # 0, 0.5, 1, ... 4
    regions = []
    for (x, y, w, h, mode, form) in rects:
        out = (torch.randn((N, C, h, w), generator=g) * 1.5).to(DTYPES[out_dn])
        aux = None
        if form == "mask":
            aux = torch.rand((h, w), generator=g)
        elif form == "4d":
            aux = torch.rand((1, 1, h, w), generator=g) * 3
        elif form == "2d":
            aux = torch.rand((h, w), generator=g) * 3
        regions.append((x, y, w, h, mode, out, aux))
    return xb, weights, regions


@gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("out_dn", list(DTYPES))
@pytest.mark.parametrize("canvas_dn", list(DTYPES))
def test_dtype_matrix(canvas_dn, out_dn, layout):
    with_weights, rects = LAYOUTS[layout]
    xb, weights, regions = _random_case(17, 2, 4, 40, 56, canvas_dn, out_dn, rects, with_weights)
    want = _check_both_entries(xb, weights, regions, f"canvas {canvas_dn} output {out_dn} {layout}", windows=[(0, 13), (13, 39), (39, 40)])
    if (canvas_dn, out_dn) in SPLITS:
        cast = [(x, y, w, h, m, o.to(xb.dtype), a) for (x, y, w, h, m, o, a) in regions]
        assert _differs(region_composite_reference(xb, weights, cast), want), "rounding the outputs first would pass unnoticed"


# ------------------------------------------------------------------------------------------------ sizes: the grid-stride loop
@gpu
@pytest.mark.parametrize("canvas_dn,out_dn", [("f16", "f32"), ("bf16", "f16"), ("f32", "bf16")])
def test_cfg2_canvas_runs_the_stride_loop_into_regions(canvas_dn, out_dn):
    """[2, 4, 512, 512] is 3.5 passes of the capped grid; the regions reach the last rows and columns of every plane, so
    the later passes land inside them."""
    N, C, H, W = 2, 4, 512, 512
    assert N * C * H * W > 2 * GRID_CAP
    rects = [(0, 0, W, H, 0, None), (300, 400, 212, 112, 1, "mask"), (17, 450, 100, 62, 0, None), (500, 0, 12, H, 1, "mask"),
             (0, H - 1, W, 1, 0, None), (128, 128, 256, 256, 1, "mask"), (511, 511, 1, 1, 1, "mask")]
    xb, weights, regions = _random_case(23, N, C, H, W, canvas_dn, out_dn, rects, True)
    _check_both_entries(xb, weights, regions, f"cfg2 {canvas_dn}/{out_dn}", windows=[(0, 1), (1, 257), (257, 511), (511, 512)])


@gpu
@pytest.mark.parametrize("shape", [(3, 5, 37, 61), (3, 5, 203, 211)], ids=["under_cap", "just_over_cap"])
def test_odd_plane_counts_and_ragged_totals(shape):
    N, C, H, W = shape
    total = N * C * H * W
    assert total % 256 != 0 and (total < GRID_CAP) == (H < 100)
    rects = [(0, 0, W, H, 0, None), (W // 3, H // 4, W - W // 3, H - H // 4, 1, "mask"), (1, H // 2, W // 2, H // 2 - 1, 0, "4d"),
             (W - 1, 0, 1, H, 1, "mask")]
    for canvas_dn, out_dn in (("f16", "f32"), ("bf16", "bf16")):
        xb, weights, regions = _random_case(total % 1000, N, C, H, W, canvas_dn, out_dn, rects, True)
        _check_both_entries(xb, weights, regions, f"{shape} {canvas_dn}/{out_dn}", windows=[(0, 5), (5, H - 2), (H - 2, H)])


# ------------------------------------------------------------------------------------------------ limits
def _stacked(n, seed, mode_of):
    """n regions that all cover pixel (x=5, y=4) of a [1, 3, 9, 11] canvas, fp32 outputs."""
    g = torch.Generator().manual_seed(seed)
    rects = []
    for k in range(n):
        x0, y0 = int(torch.randint(0, 6, (1,), generator=g)), int(torch.randint(0, 5, (1,), generator=g))
        w, h = int(torch.randint(6 - x0, 12 - x0, (1,), generator=g)), int(torch.randint(5 - y0, 10 - y0, (1,), generator=g))
        rects.append((x0, y0, w, h, mode_of(k), "mask" if mode_of(k) == 1 else None))
    return _random_case(seed, 1, 3, 9, 11, "f16", "f32", rects, True)


@gpu
@pytest.mark.parametrize("n", [16, 32])
@pytest.mark.parametrize("modes", ["background", "foreground", "mixed"])
def test_regions_stacked_over_one_pixel(n, modes):
    mode_of = {"background": lambda k: 0, "foreground": lambda k: 1, "mixed": lambda k: k % 2}[modes]
    xb, weights, regions = _stacked(n, n + len(modes), mode_of)
    assert all(x <= 5 < x + w and y <= 4 < y + h for (x, y, w, h, *_rest) in regions)
    for with_weights in (True, False):
        _check_both_entries(xb, weights if with_weights else None, regions, f"{n} {modes} weights={with_weights}",
                            windows=[(0, 4), (4, 5), (5, 9)])


def _raw_table(regions):
    from multidiffusion_upscaler_for_automatic1111_b200._cabi import TdRegion, dtype_code
    arr = (TdRegion * max(1, len(regions)))()
    for i, (x, y, w, h, m, o, a) in enumerate(regions):
        arr[i] = TdRegion(x, y, w, h, m, dtype_code(o.dtype), o.data_ptr(), None if a is None else a.data_ptr())
    return arr


@gpu
def test_33_regions_are_unsupported_and_out_untouched():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi, engine
    xb, weights, regions = _stacked(33, 5, lambda k: k % 2)
    regions = [(x, y, w, h, m, o, None if a is None else a.contiguous()) for (x, y, w, h, m, o, a) in _cuda(regions)]
    xd, wd = xb.cuda(), weights.cuda()
    arr = _raw_table(regions)
    N, C, H, W = xb.shape
    for rows in (None, (0, H), (4, 5)):
        out = torch.full((N, C, H, W), float("nan"), device="cuda")
        st = _cabi.current_stream_ptr()
        if rows is None:
            status = _cabi.lib.td_region_composite(xd.data_ptr(), wd.data_ptr(), arr, 33, N, C, H, W, _cabi.TD_F16, out.data_ptr(), st)
        else:
            status = _cabi.lib.td_region_composite_rows(xd.data_ptr(), wd.data_ptr(), arr, 33, N, C, H, W, _cabi.TD_F16, out.data_ptr(),
                                                       rows[0], rows[1], st)
        torch.cuda.synchronize()
        assert status == _cabi.TD_ERR_UNSUPPORTED and b"TD_MAX_REGIONS" in _cabi.lib.td_last_error(), rows
        assert bool(out.isnan().all()), f"{rows}: a refused call wrote into out"
    with pytest.raises(_cabi.TdError) as e:
        engine.region_composite(xd, wd, regions)
    assert e.value.status == _cabi.TD_ERR_UNSUPPORTED
    # 32 of them still run
    _same(engine.region_composite(xd, wd, regions[:32]).cpu(), region_composite_reference(xb, weights, regions[:32]), "first 32")


# ------------------------------------------------------------------------------------------------ geometry edges
GEOMETRY = {   # name: ((N, C, H, W), [(x, y, w, h, mode)])
    "one_pixel_regions": ((1, 2, 8, 10), [(0, 0, 1, 1, 0), (9, 7, 1, 1, 1), (4, 3, 1, 1, 1), (4, 3, 1, 1, 0), (9, 0, 1, 1, 1)]),
    "one_row_and_one_column": ((2, 1, 8, 10), [(0, 3, 10, 1, 0), (6, 0, 1, 8, 1), (0, 7, 10, 1, 1), (9, 0, 1, 8, 0)]),
    "region_is_the_canvas": ((1, 3, 7, 9), [(0, 0, 9, 7, 1), (0, 0, 9, 7, 0), (0, 0, 9, 7, 1)]),
    "ending_at_W_and_H": ((1, 2, 11, 13), [(8, 7, 5, 4, 0), (10, 2, 3, 9, 1), (0, 10, 13, 1, 1), (12, 10, 1, 1, 0)]),
    "W_is_1": ((2, 2, 9, 1), [(0, 0, 1, 9, 0), (0, 4, 1, 3, 1), (0, 8, 1, 1, 1)]),
    "H_is_1": ((1, 3, 1, 13), [(0, 0, 13, 1, 1), (5, 0, 3, 1, 0), (12, 0, 1, 1, 1)]),
    "odd_W": ((1, 1, 6, 37), [(3, 1, 31, 4, 1), (0, 0, 37, 6, 0), (36, 5, 1, 1, 1), (1, 0, 35, 1, 0)]),
    "one_pixel_canvas": ((1, 4, 1, 1), [(0, 0, 1, 1, 0), (0, 0, 1, 1, 1), (0, 0, 1, 1, 1)]),
}


@gpu
@pytest.mark.parametrize("name", list(GEOMETRY))
@pytest.mark.parametrize("canvas_dn,out_dn", [("f16", "f32"), ("bf16", "bf16"), ("f32", "f16")])
def test_geometry_edges(name, canvas_dn, out_dn):
    (N, C, H, W), rects = GEOMETRY[name]
    for with_weights in (True, False):
        full = [(x, y, w, h, m, "mask" if m == 1 else (None if with_weights else "2d")) for (x, y, w, h, m) in rects]
        xb, weights, regions = _random_case(len(name), N, C, H, W, canvas_dn, out_dn, full, with_weights)
        _check_both_entries(xb, weights, regions, f"{name} {canvas_dn}/{out_dn} weights={with_weights}")


@gpu
def test_rows_windows_on_a_ragged_canvas():
    """Windows [0,0), [H-1,H), one middle row, and ones whose lengths are not multiples of 8."""
    rects = [(0, 0, 37, 21, 0, None), (3, 2, 30, 17, 1, "mask"), (20, 10, 17, 11, 1, "mask"), (5, 20, 9, 1, 0, None)]
    xb, weights, regions = _random_case(3, 2, 3, 21, 37, "f16", "f32", rects, True)
    _check_both_entries(xb, weights, regions, "ragged windows", windows=[(0, 0), (20, 21), (10, 11), (1, 10), (11, 20), (21, 21)])


# ------------------------------------------------------------------------------------------------ refusals
@gpu
def test_invalid_arguments_are_refused_with_out_untouched():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    N, C, H, W = 1, 2, 8, 12
    xb = torch.randn((N, C, H, W)).half().cuda()
    weights = torch.ones((H, W), device="cuda")
    good = [(2, 1, 6, 5, 0, torch.randn((N, C, 5, 6), device="cuda"), None),
            (4, 3, 8, 5, 1, torch.randn((N, C, 5, 8), device="cuda").half(), torch.rand((5, 8), device="cuda"))]
    lib, st = _cabi.lib, _cabi.current_stream_ptr()
    region_cases = {"x<0": ("x", -1), "y<0": ("y", -1), "w=0": ("w", 0), "w<0": ("w", -3), "h=0": ("h", 0), "h<0": ("h", -2),
                    "x+w>W": ("x", W - 5), "y+h>H": ("y", H - 4), "null out": ("out", None), "mode 2": ("mode", 2),
                    "mode -1": ("mode", -1), "foreground without mask": ("aux", None), "dtype 3": ("dtype", 3), "dtype -1": ("dtype", -1)}

    def call(entry, arr, n, xp, N_, C_, H_, W_, dt, outp):
        if entry == "whole":
            return lib.td_region_composite(xp, weights.data_ptr(), arr, n, N_, C_, H_, W_, dt, outp, st)
        return lib.td_region_composite_rows(xp, weights.data_ptr(), arr, n, N_, C_, H_, W_, dt, outp, 0, H, st)

    for entry in ("whole", "rows"):
        out = torch.full((N, C, H, W), float("nan"), device="cuda")
        assert call(entry, _raw_table(good), 2, xb.data_ptr(), N, C, H, W, _cabi.TD_F16, out.data_ptr()) == _cabi.TD_OK
        assert not bool(out.isnan().any())
        refused = []
        for what, (field, value) in region_cases.items():
            arr = _raw_table(good)
            setattr(arr[1], field, value)          # the second region: the first is valid and must not be half-applied
            refused.append((what, arr, 2, xb.data_ptr(), N, C, H, W, _cabi.TD_F16))
        refused += [("null x_buffer", _raw_table(good), 2, None, N, C, H, W, _cabi.TD_F16),
                    ("negative n_regions", _raw_table(good), -1, xb.data_ptr(), N, C, H, W, _cabi.TD_F16),
                    ("null regions", None, 2, xb.data_ptr(), N, C, H, W, _cabi.TD_F16),
                    ("dtype 3", _raw_table(good), 2, xb.data_ptr(), N, C, H, W, 3),
                    ("dtype -1", _raw_table(good), 2, xb.data_ptr(), N, C, H, W, -1)]
        for k, what in enumerate("NCHW"):
            for bad in (0, -1):
                dims = [N, C, H, W]
                dims[k] = bad
                refused.append((f"{what}={bad}", _raw_table(good), 2, xb.data_ptr(), *dims, _cabi.TD_F16))
        for (what, arr, n, xp, N_, C_, H_, W_, dt) in refused:
            out = torch.full((N, C, H, W), float("nan"), device="cuda")
            status = call(entry, arr, n, xp, N_, C_, H_, W_, dt, out.data_ptr())
            torch.cuda.synchronize()
            assert status == _cabi.TD_ERR_INVALID_ARG, f"{entry} {what}: status {status}"
            assert bool(out.isnan().all()), f"{entry} {what}: a refused call wrote into out"
        assert call(entry, _raw_table(good), 2, xb.data_ptr(), N, C, H, W, _cabi.TD_F16, None) == _cabi.TD_ERR_INVALID_ARG, "null out"


@gpu
def test_engine_refuses_bad_shapes_and_host_tensors():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    xb = torch.zeros((1, 4, 16, 16), device="cuda", dtype=torch.float16)
    out_ok = torch.zeros((1, 4, 5, 6), device="cuda")
    for bad in ((1, 4, 6, 5), (1, 3, 5, 6), (2, 4, 5, 6)):
        with pytest.raises(ValueError, match="output shape"):
            engine.region_composite(xb, None, [(0, 0, 6, 5, 0, torch.zeros(bad, device="cuda"), None)])
        with pytest.raises(ValueError, match="output shape"):
            engine.region_composite_rows(xb, None, [(0, 0, 6, 5, 0, torch.zeros(bad, device="cuda"), None)], 0, 16,
                                         torch.zeros((1, 4, 16, 16), device="cuda"))
    with pytest.raises(RuntimeError, match="CUDA"):
        engine.region_composite(xb.cpu(), None, [])
    with pytest.raises(RuntimeError, match="CUDA"):
        engine.region_composite(xb, None, [(0, 0, 6, 5, 0, out_ok.cpu(), None)])
    with pytest.raises(RuntimeError, match="CUDA"):
        engine.region_composite_rows(xb.cpu(), None, [], 0, 16, torch.zeros((1, 4, 16, 16)))


# ------------------------------------------------------------------------------------------------ the delegates
_K = torch.tensor(0.7071, dtype=torch.float32)      # fp32 UNet stand-ins: outputs with more bits than the latent


def _f32_denoise(t, bb, N):
    return synth.fake_denoise(t.float(), bb, N) * _K.to(t.device)


def _f32_region_denoise(t, j):
    return synth.fake_region_denoise(t.float(), j) * _K.to(t.device)


def _delegate_step(method, x, rows):
    import types

    from multidiffusion_upscaler_for_automatic1111_b200 import MixtureOfDiffusers, MultiDiffusion, host
    G = REGION_GRID
    N = x.shape[0]
    p = types.SimpleNamespace(width=G["W"] * 8, height=G["H"] * 8, sampler_name="Euler a", disable_extra_networks=True, batch_size=1,
                              steps=20, styles=None, all_prompts=["a photo"], all_negative_prompts=["blurry"])
    sampler = types.SimpleNamespace(model_wrap_cfg=types.SimpleNamespace(inner_model=types.SimpleNamespace(forward=None),
                                                                         image_cfg_scale=None, step=0))
    d = (MultiDiffusion if method == "md" else MixtureOfDiffusers)(p, sampler)
    d.init_grid_bbox(G["tw"], G["th"], G["ov"], G["bs"])
    d.init_custom_bbox({i: row for i, row in enumerate(rows)}, True, False)
    d.init_done()
    if method == "md":
        return d.sample_one_step(x, None, lambda t, bb: _f32_denoise(t, bb, N), lambda t, j, b: _f32_region_denoise(t, j))
    it = {"i": 0}

    def apply_model(x_tile, t, c):
        bb = d.batched_bboxes[it["i"]]
        it["i"] += 1
        return _f32_denoise(x_tile, bb, N)
    model = types.SimpleNamespace(apply_model=apply_model, cond_stage_key="txt", model=types.SimpleNamespace(conditioning_key="crossattn"))
    host.use_shared(types.SimpleNamespace(state=types.SimpleNamespace(interrupted=False, sampling_step=0, sampling_steps=1), sd_model=model))
    try:
        d.custom_apply_model = lambda x_tile, t, c, bbox_id, bbox: _f32_region_denoise(x_tile, bbox_id)
        d.hook()
        cond = {"c_crossattn": [torch.zeros(N, 2, 4, device=x.device)], "c_concat": [torch.zeros(N, 5, 1, 1, device=x.device)]}
        out = model.apply_model(x, torch.ones(N, device=x.device), cond).clone()
        d.unhook()
        return out
    finally:
        host.use_shared(None)


def _oracle_step(method, x, rows, region_denoise):
    G = REGION_GRID
    N = x.shape[0]
    plan = tiling.GridPlan(G["W"], G["H"], G["tw"], G["th"], G["ov"], G["bs"], method == "mod")
    regs = region.make_regions(rows, G["W"], G["H"])
    w = region.weights_with_regions(plan.weights, regs, G["H"], G["W"], method)
    den = lambda t, bb: _f32_denoise(t, bb, N)
    if method == "md":
        return region.multidiffusion_region_step(x, plan.batched_bboxes, w, regs, den, region_denoise, True)
    return region.mixture_region_step(x, plan.batched_bboxes, plan.tile_weights, w, regs, den, region_denoise, True)


@gpu
@pytest.mark.parametrize("method", ["md", "mod"])
@pytest.mark.parametrize("dn", ["f16", "bf16"])
def test_delegate_region_step_with_fp32_unet_outputs(method, dn):
    """One MultiDiffusion / Mixture of Diffusers step with BACKGROUND and FOREGROUND regions on the real kernels, the UNet
    returning fp32 for an fp16 / bf16 latent: the oracle's region pass rounds each add once."""
    rows = REGION_CASES[0][2]
    x = synth.latent(77, (REGION_GRID["N"], REGION_GRID["C"], REGION_GRID["H"], REGION_GRID["W"]), DTYPES[dn])
    want = _oracle_step(method, x, rows, _f32_region_denoise)
    rounded = _oracle_step(method, x, rows, lambda t, j: _f32_region_denoise(t, j).to(t.dtype))
    assert _differs(rounded.float(), want.float()), "rounding the region outputs first would pass unnoticed"
    got = _delegate_step(method, x.cuda(), rows).cpu()
    _same(got, want, f"{method} {dn} delegate, fp32 UNet")
