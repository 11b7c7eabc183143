"""TEST INFRASTRUCTURE -- oracle for DemoFusion's per-step tile path (torch-CPU restatement of
tile_methods/demofusion.py:219-324; `jitter_range` > 0 = random-jitter mode on the zero-padded latent).

  local windows   :254-264   scatter, per-tile add in x.dtype, exact fp32 COUNT, x_local = (buffer / count) rounded to x.dtype
  gaussian filter :164-178   depthwise conv, kernel 2s-1, sigma = sig * c3, kernel cast to x.dtype
  renormalise     :269-273   (g - g.mean()) / g.std() * x.std() + x.mean()   (unbiased std, every op in x.dtype)
  global views    :283-310   s*s dilated views x[:, :, by::s, bx::s] (mixture: raw views then blurred views, /2)
  mix             :312-324   x_local * (1 - c2) + x_global * c2
Quirk kept: the strided slices stop at `end = W - jitter_range` for BOTH axes (:280).
Deliberate difference: the reference counts the windows in x.dtype (`torch.zeros_like(x_in)`, `+= 1`).  A half-precision
count stops growing at 256 (bf16) or 2048 (fp16), where + 1 rounds back, and would scale x_local by up to coverage / 256;
the reference escapes this only because the WebUI samples in fp32, where the count is exact up to 2^24.  The count here is
fp32 (exact), as the kernels count; below those two limits both rules give the same bits.

Random jitter: the caller pads x_in by jitter_range (:204), the local windows come in padded coordinates
(tiling.demofusion_views_jitter), the dilated views start at jitter_range + (bx, by) and the caller crops.
"""
from __future__ import annotations

import math
from typing import Callable, List, Sequence, Tuple

import torch
import torch.nn.functional as F

BBox = Tuple[int, int, int, int]


def cosine_factor(current_step: int, t_enc: int) -> torch.Tensor:
    """demofusion.py:194 -- a 0-dim fp32 CPU tensor, exactly as the reference builds it."""
    return 0.5 * (1 + torch.cos(torch.pi * torch.tensor(((current_step + 1) / (t_enc + 1)))))


def gaussian_kernel(kernel_size: int, sigma, channels: int) -> torch.Tensor:
    """demofusion.py:164-171 (fp32)."""
    x_coord = torch.arange(kernel_size)
    g1 = torch.exp(-(x_coord - (kernel_size - 1) / 2) ** 2 / (2 * sigma ** 2))
    g1 = g1 / g1.sum()
    g2 = g1[:, None] * g1[None, :]
    return g2[None, None, :, :].repeat(channels, 1, 1, 1)


def gaussian_filter(latents: torch.Tensor, kernel_size: int, sigma) -> torch.Tensor:
    """demofusion.py:173-178."""
    channels = latents.shape[1]
    kernel = gaussian_kernel(kernel_size, sigma, channels).to(latents.dtype)
    if latents.dtype in (torch.float16, torch.bfloat16):   # CPU conv in half is not everywhere available: fp32 accumulate
        return F.conv2d(latents.float(), kernel.float(), padding=kernel_size // 2, groups=channels).to(latents.dtype)
    return F.conv2d(latents, kernel, padding=kernel_size // 2, groups=channels)


def global_views(scale: int, mixture: bool) -> List[Tuple[int, int]]:
    """demofusion.py:87-99: (x, y) offsets, row-major; doubled in mixture mode."""
    views = [(col, row) for row in range(scale) for col in range(scale)]
    return views + views if mixture else views


def local_blend(x_like: torch.Tensor, windows: Sequence[BBox], outs: Sequence[torch.Tensor]) -> torch.Tensor:
    """demofusion.py:259-264 for windows (x, y, w, h) inside the canvas of x_like [N,C,H,W] and their outputs outs[t]
    [N,C,h,w], in list order: the buffer accumulated window by window in x_like.dtype, divided by the exact fp32 count of
    the windows covering each pixel (1 where none does).  Returns that fp32 quotient (x_local is it rounded to x.dtype),
    on x_like's device."""
    assert len(windows) == len(outs)
    x_buffer = torch.zeros_like(x_like)
    count = torch.zeros(x_like.shape[2:], dtype=torch.float32, device=x_like.device)
    for (x, y, w, h), out in zip(windows, outs):
        x_buffer[:, :, y:y + h, x:x + w] += out
        count[y:y + h, x:x + w] += 1
    return x_buffer.float() / torch.where(count == 0, 1.0, count)


def sample_one_step(x_in: torch.Tensor, local_batches: Sequence[Sequence[BBox]], global_batches: Sequence[Sequence[Tuple[int, int]]],
                    scale: int, mixture: bool, use_gaussian: bool, sig: float, cos_factor: torch.Tensor, cs2: float, cs3: float,
                    denoise_local: Callable, denoise_global: Callable, jitter_range: int = 0) -> torch.Tensor:
    """demofusion.py:219-324.  denoise_*(x_tile, views) stand for the UNet."""
    N = x_in.shape[0]
    dt = x_in.dtype
    windows, outs = [], []
    for bboxes in local_batches:
        x_tile = torch.cat([x_in[:, :, y:y + h, x:x + w] for (x, y, w, h) in bboxes], dim=0)
        out = denoise_local(x_tile, bboxes)
        windows += list(bboxes)
        outs += [out[i * N:(i + 1) * N] for i in range(len(bboxes))]
    x_local = local_blend(x_in, windows, outs).to(dt)

    x_buffer = torch.zeros_like(x_in)
    weights = torch.zeros_like(x_in)
    std_, mean_ = x_in.std(), x_in.mean()
    c3 = 0.99 * cos_factor ** cs3 + 1e-2
    x_in_g = None
    if use_gaussian:
        x_in_g = gaussian_filter(x_in, kernel_size=2 * scale - 1, sigma=sig * c3)
        x_in_g = (x_in_g - x_in_g.mean()) / x_in_g.std() * std_ + mean_

    x_global = torch.zeros_like(x_local)
    jr = jitter_range
    end = x_global.shape[3] - jr
    total = sum(len(b) for b in global_batches)
    seen = 0
    for views in global_batches:
        srcs = []
        for (bx, by) in views:
            src = x_in if (mixture and seen < total // 2) else x_in_g
            srcs.append(src[:, :, by + jr:end:scale, bx + jr:end:scale])
            seen += 1
        out = denoise_global(torch.cat(srcs, dim=0), views)
        for idx, (bx, by) in enumerate(views):
            x_global[:, :, by + jr:end:scale, bx + jr:end:scale] += out[idx * N:(idx + 1) * N]
    if mixture:
        x_buffer += x_global / 2
    else:
        x_buffer += x_global
    weights += 1
    x_global = x_buffer / weights
    c2 = cos_factor ** cs2
    return x_local * (1 - c2) + x_global * c2
