"""DemoFusion's local-window blend without a GPU: the rules tests/test_gpu_zz_demofusion_windows.py holds the device to.

  engine._fit_batch_table    more than 128 window batches fold into at most 128 tensors, tile order kept, and the fitted
                             (num_batches, tile_bs) passes the C entries' rule (nb - 1) * tile_bs < T <= nb * tile_bs
  C-entry refusals           129 batch pointers, inconsistent tile_bs / num_batches, a null batch, an origin out of range:
                             refused before any launch by td_blend_bboxes(_wrap) and td_scatter_bboxes(_wrap)
  the window count           the host emulation of the blend body (tests/emul/jitter_host_emul.cu) at coverage 1024 in
                             bf16 and 4096 in fp16 equals the oracles' local blend, whose count is exact; up to coverage
                             256 (bf16) / 2048 (fp16) that blend equals the reference's x.dtype count bit for bit, one
                             window past it it does not
"""
import ctypes

import numpy as np
import pytest
import torch

import demofusion_wrap_oracle as dwo
import wrap_oracle as wo
from helpers import DTYPES
from oracle import demofusion as odf
from oracle import synth
from test_jitter_emulation import CODE, emul  # noqa: F401  (module fixture: the host emulation library)

TD_MAX_BATCH_PTRS = 128


def _cabi():
    from multidiffusion_upscaler_for_automatic1111_b200 import _cabi
    return _cabi


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


# ------------------------------------------------------------------------------------------------ batch-table fit
@pytest.mark.parametrize("nb", [129, 257, 1089])
@pytest.mark.parametrize("tile_bs", [1, 3, 8])
def test_fit_batch_table_folds_past_128_batches_in_tile_order(nb, tile_bs):
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    N = 2
    T = (nb - 1) * tile_bs + max(1, tile_bs - 1)           # the last batch is partial whenever tile_bs > 1
    rows = torch.arange(T * N, dtype=torch.float32).view(T * N, 1, 1, 1)
    batches = [rows[b * tile_bs * N:min((b + 1) * tile_bs, T) * N] for b in range(nb)]
    fitted, bs = engine._fit_batch_table(None, batches, tile_bs)
    assert len(fitted) <= TD_MAX_BATCH_PTRS
    assert bs % tile_bs == 0 and (len(fitted) - 1) * bs < T <= len(fitted) * bs
    for b, t in enumerate(fitted):
        assert t.shape[0] == min(bs, T - b * bs) * N
    assert torch.equal(torch.cat(fitted), rows)


def test_fit_batch_table_keeps_128_batches_as_they_are():
    from multidiffusion_upscaler_for_automatic1111_b200 import engine
    batches = [torch.full((3, 1, 1, 1), float(b)) for b in range(TD_MAX_BATCH_PTRS)]
    fitted, bs = engine._fit_batch_table(None, batches, 3)
    assert bs == 3 and all(a is b for a, b in zip(fitted, batches))


# ------------------------------------------------------------------------------------------------ C-entry refusals
H, W, TH, TW, N, C = 20, 30, 8, 12, 1, 2


def _scratch(nbytes=1 << 16):
    return torch.zeros(nbytes, dtype=torch.uint8, device="cuda" if torch.cuda.is_available() else "cpu")


def _org(*xy):
    return (ctypes.c_int32 * len(xy))(*xy)


def _blend(entry, nb, tile_bs, T, origins, buf, null_at=None, wrap=3):
    """td_blend_bboxes or td_blend_bboxes_wrap on a scratch buffer: every pointer is valid for a launch of these sizes."""
    cabi = _cabi()
    ptrs = (ctypes.c_void_p * max(nb, 1))(*([buf.data_ptr()] * max(nb, 1)))
    if null_at is not None:
        ptrs[null_at] = None
    out = ctypes.cast(ctypes.c_void_p(buf.data_ptr() + buf.numel() // 2), ctypes.POINTER(ctypes.c_float))
    stream = cabi.current_stream_ptr() if torch.cuda.is_available() else None
    if entry == "td_blend_bboxes":
        return cabi.lib.td_blend_bboxes(ptrs, nb, tile_bs, buf.data_ptr(), origins, T, N, C, H, W, TH, TW, cabi.TD_F16, out, stream)
    return cabi.lib.td_blend_bboxes_wrap(ptrs, nb, tile_bs, buf.data_ptr(), origins, T, N, C, H, W, TH, TW, wrap, cabi.TD_F16, out, stream)


def _scatter(entry, T, origins, buf, wrap=3):
    cabi = _cabi()
    stream = cabi.current_stream_ptr() if torch.cuda.is_available() else None
    tiles = buf.data_ptr() + buf.numel() // 2
    if entry == "td_scatter_bboxes":
        return cabi.lib.td_scatter_bboxes(buf.data_ptr(), tiles, buf.data_ptr(), origins, T, N, C, H, W, TH, TW, cabi.TD_F16, stream)
    return cabi.lib.td_scatter_bboxes_wrap(buf.data_ptr(), tiles, buf.data_ptr(), origins, T, N, C, H, W, TH, TW, wrap, cabi.TD_F16, stream)


BLENDS = ["td_blend_bboxes", "td_blend_bboxes_wrap"]


def _refused(st, name, what=None):
    msg = _cabi().lib.td_last_error().decode()
    assert st == _cabi().TD_ERR_INVALID_ARG, f"{name}: status {st} ({msg})"
    assert msg.startswith(name + ":"), msg
    if what is not None:
        assert what in msg, msg


@pytest.mark.parametrize("entry", BLENDS)
def test_blend_entries_refuse_129_batch_pointers(entry):
    buf = _scratch()
    T = TD_MAX_BATCH_PTRS + 1
    _refused(_blend(entry, T, 1, T, _org(*([0, 0] * T)), buf), entry, "bad arguments")
    # the folded table of engine.blend_bboxes: 65 batches of 2 for the same 129 windows
    st = _blend(entry, 65, 2, T, _org(*([0, 0] * T)), buf)
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        assert st == _cabi().TD_OK
    else:
        assert st == _cabi().TD_ERR_CUDA          # every check passed; only the launch itself fails without a device


@pytest.mark.parametrize("entry", BLENDS)
@pytest.mark.parametrize("nb,tile_bs,T", [(3, 4, 13), (4, 4, 12), (2, 4, 4), (0, 4, 1), (1, 0, 1), (1, 1, 0), (2, -1, 1)],
                         ids=["too_few", "one_too_many", "empty_last", "no_batch", "tile_bs0", "no_window", "tile_bs_negative"])
def test_blend_entries_refuse_inconsistent_batch_tables(entry, nb, tile_bs, T):
    buf = _scratch()
    _refused(_blend(entry, nb, tile_bs, T, _org(*([0, 0] * max(T, 1))), buf), entry, "bad arguments")


@pytest.mark.parametrize("entry", BLENDS)
@pytest.mark.parametrize("null_at", [0, 2])
def test_blend_entries_refuse_a_null_batch(entry, null_at):
    buf = _scratch()
    _refused(_blend(entry, 3, 2, 6, _org(*([0, 0] * 6)), buf, null_at=null_at), entry, f"null batch {null_at}")


# bounded entries: 0 <= o and o + tile <= L.  Wrap entries, per mode: wrapped axis 0 <= o < L, bounded -(tile-1) <= o <= L-1
BAD_BOUNDED = [(-1, 0), (0, -1), (W - TW + 1, 0), (0, H - TH + 1), (1 << 30, 0)]
BAD_WRAP = {1: [(-1, 0), (W, 0), (0, -TH), (0, H)], 2: [(-TW, 0), (W, 0), (0, -1), (0, H)], 3: [(-1, 0), (W, 0), (0, -1), (0, H)]}


@pytest.mark.parametrize("kind", ["scatter", "blend"])
def test_bounded_list_entries_refuse_origins_off_the_canvas(kind):
    buf = _scratch()
    for ox, oy in BAD_BOUNDED:
        origins = _org(0, 0, ox, oy)
        if kind == "scatter":
            _refused(_scatter("td_scatter_bboxes", 2, origins, buf), "td_scatter_bboxes", "leaves")
        else:
            _refused(_blend("td_blend_bboxes", 1, 2, 2, origins, buf), "td_blend_bboxes", "leaves")


@pytest.mark.parametrize("kind", ["scatter", "blend"])
@pytest.mark.parametrize("wrap", [1, 2, 3], ids=["x", "y", "xy"])
def test_wrap_list_entries_refuse_origins_out_of_range(kind, wrap):
    buf = _scratch()
    for ox, oy in BAD_WRAP[wrap]:
        origins = _org(0, 0, ox, oy)
        if kind == "scatter":
            _refused(_scatter("td_scatter_bboxes_wrap", 2, origins, buf, wrap), "td_scatter_bboxes_wrap", "out of range")
        else:
            _refused(_blend("td_blend_bboxes_wrap", 1, 2, 2, origins, buf, wrap=wrap), "td_blend_bboxes_wrap", "out of range")


# ------------------------------------------------------------------------------------------------ the window count
def stacked_windows(cov_x, cov_y, tw, th, wrap, L_x, L_y):
    """cov_x * cov_y windows of tw x th at unit stride, row-major: the pixel at (cov_x - 1, cov_y - 1) past the first origin
    is covered by all of them.  On a wrapped axis the origins start half a window before the seam."""
    x0 = L_x - tw // 2 if wrap & wo.WRAP_X else 0
    y0 = L_y - th // 2 if wrap & wo.WRAP_Y else 0
    return [((x0 + i) % L_x, (y0 + j) % L_y, tw, th) for j in range(cov_y) for i in range(cov_x)]


def saturating_blend(x_like, windows, outs, wrap):
    """The reference's rule: buffer AND count in x.dtype (`zeros_like(x_in)`, `+= 1`), quotient in x.dtype."""
    Hc, Wc = x_like.shape[2], x_like.shape[3]
    buf, cnt = torch.zeros_like(x_like), torch.zeros_like(x_like)
    for b, out in zip(windows, outs):
        iy, oky = dwo.axis_indices(b[1], b[3], Hc, bool(wrap & wo.WRAP_Y))
        ix, okx = dwo.axis_indices(b[0], b[2], Wc, bool(wrap & wo.WRAP_X))
        idx = (slice(None), slice(None), iy[oky][:, None], ix[okx][None, :])
        buf[idx] = buf[idx] + out[:, :, oky][:, :, :, okx]
        cnt[idx] = cnt[idx] + 1
    return buf / torch.where(cnt == 0, torch.tensor(1, dtype=x_like.dtype), cnt)


def fixed_blend(x_like, windows, outs, wrap):
    """The oracles' local blend: oracle/demofusion.py's on a bounded canvas, demofusion_wrap_oracle's on a periodic one."""
    if wrap:
        return dwo.local_blend(x_like, windows, outs, wrap)
    return odf.local_blend(x_like, windows, outs)


SATURATION = {"bf16": 256, "f16": 2048}


@pytest.mark.parametrize("wrap", [0, 3], ids=["bounded", "wrap_xy"])
@pytest.mark.parametrize("dn", list(SATURATION))
def test_exact_count_equals_the_dtype_count_up_to_its_saturation(dn, wrap):
    """At coverage 256 (bf16) / 2048 (fp16) the fixed oracles equal the reference's x.dtype count bit for bit; one more
    window over the fully covered pixel, and the dtype count (+ 1 rounds back) gives another quotient there."""
    dt, sat = DTYPES[dn], SATURATION[dn]
    cx, cy = (16, 16) if sat == 256 else (64, 32)
    tw, th = cx, cy
    Lx, Ly = 2 * cx + 3, 2 * cy + 5
    x = torch.zeros((1, 2, Ly, Lx), dtype=dt)
    windows = stacked_windows(cx, cy, tw, th, wrap, Lx, Ly)
    assert len(windows) == sat
    outs = [synth.latent(500 + t, (1, 2, th, tw), dt) for t in range(sat)]
    got = fixed_blend(x, windows, outs, wrap).to(dt)
    assert torch.equal(_bits(got), _bits(saturating_blend(x, windows, outs, wrap)))
    assert torch.equal(_bits(got), _bits(dwo.local_blend(x, windows, outs, wrap).to(dt)))      # the two oracles agree

    windows.append(windows[0])
    outs.append(torch.full((1, 2, th, tw), 3.0, dtype=dt))
    got = fixed_blend(x, windows, outs, wrap).to(dt)
    old = saturating_blend(x, windows, outs, wrap)
    last = windows[-1]
    px, py = (last[0] + cx - 1) % Lx, (last[1] + cy - 1) % Ly         # covered sat + 1 times
    assert not torch.equal(got[:, :, py, px], old[:, :, py, px])


@pytest.mark.parametrize("wrap", [0, 3], ids=["bounded", "wrap_xy"])
@pytest.mark.parametrize("dn,cov", [("bf16", 32), ("f16", 64)], ids=["bf16_coverage_1024", "f16_coverage_4096"])
def test_emulated_blend_past_the_half_counts_equals_the_fixed_oracle(emul, dn, cov, wrap):
    """cov^2 windows of cov x cov over one pixel (1024 in bf16, 4096 in fp16; 32 / 64 batches): the host run of the
    kernel's element body equals the oracle's fp32 quotient bit for bit, and the reference's saturating count does not."""
    dt = DTYPES[dn]
    Nn, Cn, L = 1, 2, 2 * cov + 3
    tile_bs = cov
    windows = stacked_windows(cov, cov, cov, cov, wrap, L, L)
    T = len(windows)
    assert T == cov * cov
    x = torch.zeros((Nn, Cn, L, L), dtype=dt)
    outs_all = synth.latent(900 + cov, (T * Nn, Cn, cov, cov), dt)
    outs = [outs_all[t * Nn:(t + 1) * Nn] for t in range(T)]
    nb = -(-T // tile_bs)
    batches = [outs_all[b * tile_bs * Nn:min((b + 1) * tile_bs, T) * Nn].contiguous() for b in range(nb)]
    ptrs = (ctypes.c_void_p * nb)(*[o.data_ptr() for o in batches])
    flat = np.array([v for b in windows for v in b[:2]], dtype=np.int32)
    got = torch.empty((Nn, Cn, L, L), dtype=torch.float32)
    if wrap:
        assert emul.td_emul_blend_bboxes_wrap(ptrs, nb, tile_bs, flat.ctypes.data_as(ctypes.c_void_p), T, Nn, Cn, L, L, cov, cov, wrap,
                                              CODE[dt], _p(got)) == 0
    else:
        emul.td_emul_blend_bboxes(ptrs, nb, tile_bs, flat.ctypes.data_as(ctypes.c_void_p), T, Nn, Cn, L, L, cov, cov, CODE[dt], _p(got))
    want = fixed_blend(x, windows, outs, wrap)
    assert torch.equal(_bits(got), _bits(want))
    assert not torch.equal(got.to(dt), saturating_blend(x, windows, outs, wrap))
