"""Oracle for seamless (periodic) DemoFusion: the local windows, jitter draws and one step on a canvas whose wrapped axes are
circles.  The reference has no periodic canvas, so these functions define the semantics the delegate and the kernels
follow; the plan rules (periodic_origins, linear_origins) are those of tests/wrap_oracle.py.

Written with explicit per-window loops and modular index arrays, with the dtype round trips of oracle/demofusion.py.
"""
from __future__ import annotations

from typing import Callable, Sequence, Tuple

import torch

from wrap_oracle import WRAP_X, WRAP_Y, BBox, linear_origins, periodic_origins


def demofusion_views(w: int, h: int, window_size: int, overlap: int, wrap: int, rng=None):
    """Seamless DemoFusion's local windows, in canvas coordinates (never padded): ([(x, y, ws, ws)] row-major, jitter_range).

    Grid: the periodic plan (periodic_origins) on a wrapped axis, the reference's split (linear_origins) on a bounded
    one, tile = window_size, overlap clamped as in demofusion.py:145.  With `rng` (Python's `random`, or a
    `random.Random`) every window is jittered, x before y, row-major, with the reference's jitter_range: on a wrapped axis
    by randint(-jr, jr) and kept mod L, on a bounded axis by the reference's border rule (demofusion.py:116-134)."""
    overlap = max(0, min(overlap, window_size - 4))
    stride = max(4, window_size - overlap)
    xs = (periodic_origins if wrap & WRAP_X else linear_origins)(w, window_size, overlap)
    ys = (periodic_origins if wrap & WRAP_Y else linear_origins)(h, window_size, overlap)
    if rng is None:
        return [(x, y, window_size, window_size) for y in ys for x in xs], 0
    jr = min(max((min(w, h) - stride) // 4, 0), min(int(window_size / 2), int(overlap / 2)))

    def draw(pos, L, wrapped):
        at_start, at_end = pos == 0, pos + window_size == L
        if wrapped or (not at_start and not at_end):
            return rng.randint(-jr, jr)
        if at_start and not at_end:
            return rng.randint(-jr, 0)
        if at_end and not at_start:
            return rng.randint(0, jr)
        return 0
    out = []
    for y in ys:
        for x in xs:
            xj = draw(x, w, bool(wrap & WRAP_X))
            yj = draw(y, h, bool(wrap & WRAP_Y))
            out.append(((x + xj) % w if wrap & WRAP_X else x + xj, (y + yj) % h if wrap & WRAP_Y else y + yj, window_size, window_size))
    return out, jr


def axis_indices(o: int, n: int, L: int, wrapped: bool):
    """Canvas indices of o .. o + n - 1 on one axis (mod L when wrapped) and which of them lie on the canvas."""
    i = torch.arange(o, o + n)
    if wrapped:
        return i % L, torch.ones(n, dtype=torch.bool)
    ok = (i >= 0) & (i < L)
    return i.clamp(0, L - 1), ok


def demofusion_crop(x: torch.Tensor, b: BBox, wrap: int) -> torch.Tensor:
    """One window of x [N,C,H,W]: modular on a wrapped axis, zeros off a bounded one."""
    H, W = x.shape[2], x.shape[3]
    iy, oky = axis_indices(b[1], b[3], H, bool(wrap & WRAP_Y))
    ix, okx = axis_indices(b[0], b[2], W, bool(wrap & WRAP_X))
    t = x[:, :, iy][:, :, :, ix].clone()
    t[:, :, ~oky] = 0
    t[:, :, :, ~okx] = 0
    return t


def demofusion_gaussian_filter(latents: torch.Tensor, kernel_size: int, sigma, wrap: int) -> torch.Tensor:
    """oracle/demofusion.gaussian_filter with circular padding on the wrapped axes (F.pad(mode="circular"), then conv2d
    zero-padding only the bounded ones); the same kernel, dtype round trips and fp32 accumulation."""
    from oracle import demofusion as odf
    F = torch.nn.functional
    channels, r = latents.shape[1], kernel_size // 2
    kernel = odf.gaussian_kernel(kernel_size, sigma, channels).to(latents.dtype)
    x = latents.float() if latents.dtype in (torch.float16, torch.bfloat16) else latents
    px, py = (r if wrap & WRAP_X else 0), (r if wrap & WRAP_Y else 0)
    if px or py:
        x = F.pad(x, (px, px, py, py), mode="circular")
    y = F.conv2d(x, kernel.to(x.dtype), padding=(0 if wrap & WRAP_Y else r, 0 if wrap & WRAP_X else r), groups=channels)
    return y.to(latents.dtype)


def demofusion_step(x: torch.Tensor, local_batches: Sequence[Sequence[BBox]], global_batches: Sequence[Sequence[Tuple[int, int]]],
                    scale: int, mixture: bool, use_gaussian: bool, sig: float, cos_factor: torch.Tensor, cs2: float, cs3: float,
                    denoise_local: Callable, denoise_global: Callable, wrap: int = 0, jitter_range: int = 0) -> torch.Tensor:
    """One DemoFusion step (demofusion.py:219-324) on the UNPADDED latent x, windows in canvas coordinates.

    wrap != 0 (seamless): windows are modular on the wrapped axes; on a bounded axis they read zeros off the canvas and
    drop those pixels in the blend.  The gaussian filter is circular on the wrapped axes, the statistics are those of x,
    and the s*s dilated views start at 0 and cover the whole canvas.
    wrap == 0 with jitter_range > 0 is the reference's padded path: x is zero-padded by jitter_range, the windows move
    by +jitter_range, the views start at jitter_range and stop at `end = W_padded - jitter_range` on both axes, and the
    result is cropped back.  Written with explicit per-window loops and modular index arrays; every op rounds in x.dtype
    where the reference's eager ops do (oracle/demofusion.py)."""
    F = torch.nn.functional
    jr = jitter_range if wrap == 0 else 0
    H0, W0 = x.shape[2], x.shape[3]
    if jr:
        x = F.pad(x, (jr, jr, jr, jr), "constant", value=0)
        local_batches = [[(bx + jr, by + jr, bw, bh) for (bx, by, bw, bh) in bb] for bb in local_batches]
    N, H, W = x.shape[0], x.shape[2], x.shape[3]
    wy, wx = bool(wrap & WRAP_Y), bool(wrap & WRAP_X)

    x_buffer = torch.zeros_like(x)
    weights = torch.zeros_like(x)
    for bboxes in local_batches:
        out = denoise_local(torch.cat([demofusion_crop(x, b, wrap) for b in bboxes], dim=0), bboxes)
        for i, b in enumerate(bboxes):
            iy, oky = axis_indices(b[1], b[3], H, wy)
            ix, okx = axis_indices(b[0], b[2], W, wx)
            idx = (slice(None), slice(None), iy[oky][:, None], ix[okx][None, :])
            x_buffer[idx] = x_buffer[idx] + out[i * N:(i + 1) * N][:, :, oky][:, :, :, okx]
            weights[idx] = weights[idx] + 1
    weights = torch.where(weights == 0, torch.tensor(1), weights)
    x_local = x_buffer / weights

    std_, mean_ = x.std(), x.mean()
    c3 = 0.99 * cos_factor ** cs3 + 1e-2
    x_in_g = None
    if use_gaussian:
        x_in_g = demofusion_gaussian_filter(x, 2 * scale - 1, sig * c3, wrap)
        x_in_g = (x_in_g - x_in_g.mean()) / x_in_g.std() * std_ + mean_

    if wrap:
        off, end_y, end_x = 0, H, W
    else:
        off, end_y, end_x = jr, min(H, W - jr), W - jr
    x_global = torch.zeros_like(x_local)
    total = sum(len(b) for b in global_batches)
    seen = 0
    for views in global_batches:
        srcs = []
        for (bx, by) in views:
            src = x if (mixture and seen < total // 2) else x_in_g
            srcs.append(src[:, :, torch.arange(off + by, end_y, scale)][:, :, :, torch.arange(off + bx, end_x, scale)])
            seen += 1
        out = denoise_global(torch.cat(srcs, dim=0), views)
        for i, (bx, by) in enumerate(views):
            idx = (slice(None), slice(None), torch.arange(off + by, end_y, scale)[:, None], torch.arange(off + bx, end_x, scale)[None, :])
            x_global[idx] = x_global[idx] + out[i * N:(i + 1) * N]
    x_global = x_global / 2 if mixture else x_global
    x_global = (torch.zeros_like(x_local) + x_global) / (torch.zeros_like(x_local) + 1)   # the reference's buffer / weights (+0 start)
    c2 = cos_factor ** cs2
    y = x_local * (1 - c2) + x_global * c2
    return y[:, :, jr:jr + H0, jr:jr + W0] if jr else y
