"""Tile bookkeeping with the reference's names (tile_utils/utils.py), computed by
the C-ABI host functions in csrc/td_host.cpp -- integer results are bit-exact with
the reference's Python float64 arithmetic.

In scope (SURVEY.md section 8 A1-A4): `BBox`, `split_bboxes`, `splitable`,
`gaussian_weights`, the `Method` / `BlendMode` enums; and for region prompt control
(section 8(f)-1): `BBoxSettings`, `build_bbox_settings`, `CustomBBox`, `feather_mask`
and the `Prompt` / `Condition` helpers (thin calls into the host's prompt parser).
`get_retouch_mask` / `NoiseInverseCache` serve tiled noise inversion (section 8(f)-3).
"""
from __future__ import annotations

import ctypes
from collections import namedtuple
from enum import Enum
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _cabi, host


class ComparableEnum(Enum):
    def __eq__(self, other: Any) -> bool:
        if isinstance(other, str):
            return self.value == other
        if isinstance(other, ComparableEnum):
            return self.value == other.value
        raise TypeError(f"unsupported type: {type(other)}")

    def __hash__(self):
        return hash(self.value)


class Method(ComparableEnum):
    MULTI_DIFF = "MultiDiffusion"
    MIX_DIFF = "Mixture of Diffusers"
    SPOT_DIFF = "SpotDiffusion"


class Method_2(ComparableEnum):
    DEMO_FU = "DemoFusion"


class BlendMode(Enum):
    FOREGROUND = "Foreground"
    BACKGROUND = "Background"


class BBox:
    """Grid bbox: `box = [x, y, x+w, y+h]`, `slicer` crops [N,C,H,W] (utils.py:69-82)."""

    __slots__ = ("x", "y", "w", "h", "box", "slicer")

    def __init__(self, x: int, y: int, w: int, h: int):
        self.x, self.y, self.w, self.h = x, y, w, h
        self.box = [x, y, x + w, y + h]
        self.slicer = (slice(None), slice(None), slice(y, y + h), slice(x, x + w))

    def __getitem__(self, idx: int) -> int:
        return self.box[idx]

    def __repr__(self):
        return f"BBox(x={self.x}, y={self.y}, w={self.w}, h={self.h})"


# one row of the region-control UI (utils.py:41-44)
BBoxSettings = namedtuple("BBoxSettings", ["enable", "x", "y", "w", "h", "prompt", "neg_prompt", "blend_mode", "feather_ratio", "seed"])
DEFAULT_BBOX_SETTINGS = BBoxSettings(False, 0.4, 0.4, 0.2, 0.2, "", "", BlendMode.BACKGROUND.value, 0.2, -1)
NUM_BBOX_PARAMS = len(BBoxSettings._fields)
NoiseInverseCache = namedtuple("NoiseInversionCache", ["model_hash", "x0", "xt", "noise_inversion_steps", "retouch", "prompts"])


def build_bbox_settings(bbox_control_states: List[Any]) -> Dict[int, BBoxSettings]:
    """Flat UI state -> {row index: BBoxSettings} (utils.py:47-65): floats rounded to 4 digits, disabled /
    degenerate rows dropped."""
    settings: Dict[int, BBoxSettings] = {}
    for index, lo in enumerate(range(0, len(bbox_control_states), NUM_BBOX_PARAMS)):
        st = BBoxSettings(*bbox_control_states[lo:lo + NUM_BBOX_PARAMS])
        st = st._replace(x=round(st.x, 4), y=round(st.y, 4), w=round(st.w, 4), h=round(st.h, 4),
                         feather_ratio=round(st.feather_ratio, 4), seed=int(st.seed))
        if not st.enable or st.x > 1.0 or st.y > 1.0 or st.w <= 0.0 or st.h <= 0.0:
            continue
        settings[index] = st
    return settings


def _float_ptr(a: np.ndarray):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def splitable(w: int, h: int, tile_w: int, tile_h: int, overlap: int = 16) -> bool:
    """utils.py:151-158; w, h in image pixels."""
    return bool(_cabi.check(_cabi.lib.td_splitable(int(w), int(h), int(tile_w), int(tile_h), int(overlap))))


def split_bboxes_xywh(w: int, h: int, tile_w: int, tile_h: int, overlap: int = 16) -> np.ndarray:
    """int32 [T,4] (x, y, w, h), row-major tile order."""
    cols, rows = ctypes.c_int(0), ctypes.c_int(0)
    n = _cabi.check(_cabi.lib.td_split_bboxes(int(w), int(h), int(tile_w), int(tile_h), int(overlap), None, 0,
                                               ctypes.byref(cols), ctypes.byref(rows)))
    out = np.empty((n, 4), dtype=np.int32)
    _cabi.check(_cabi.lib.td_split_bboxes(int(w), int(h), int(tile_w), int(tile_h), int(overlap),
                                          out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), n, None, None))
    return out


def split_bboxes(w: int, h: int, tile_w: int, tile_h: int, overlap: int = 16,
                 init_weight: Union[torch.Tensor, float] = 1.0) -> Tuple[List[BBox], torch.Tensor]:
    """utils.py:160-177: tile list + fp32 weight canvas [1,1,h,w] (`+= init_weight` per tile, list order)."""
    xywh = split_bboxes_xywh(w, h, tile_w, tile_h, overlap)
    bboxes = [BBox(int(x), int(y), int(bw), int(bh)) for x, y, bw, bh in xywh]
    weight = np.zeros((h, w), dtype=np.float32)
    if isinstance(init_weight, torch.Tensor):
        iw = init_weight.detach().to("cpu", torch.float32).numpy()
    else:
        iw = np.float32(init_weight)
    for b in bboxes:
        weight[b.y:b.y + b.h, b.x:b.x + b.w] += iw
    return bboxes, torch.from_numpy(weight).view(1, 1, h, w).to(host.device())


def gaussian_weights_np(tile_w: int, tile_h: int) -> np.ndarray:
    out = np.empty((tile_h, tile_w), dtype=np.float32)
    _cabi.check(_cabi.lib.td_gaussian_weights(int(tile_w), int(tile_h), _float_ptr(out)))
    return out


def gaussian_weights(tile_w: int, tile_h: int) -> torch.Tensor:
    """utils.py:180-194: fp32 [tile_h, tile_w] on the device (asymmetric y midpoint kept)."""
    return torch.from_numpy(gaussian_weights_np(tile_w, tile_h)).to(host.device())


def null_decorator(fn):
    return fn


keep_signature = null_decorator
controlnet = null_decorator
stablesr = null_decorator
grid_bbox = null_decorator
custom_bbox = null_decorator
noise_inverse = null_decorator


def feather_mask_np(w: int, h: int, ratio: float) -> np.ndarray:
    out = np.empty((h, w), dtype=np.float32)
    _cabi.check(_cabi.lib.td_feather_mask(int(w), int(h), float(ratio), _float_ptr(out)))
    return out


def feather_mask(w: int, h: int, ratio: float) -> torch.Tensor:
    """utils.py:196-214: fp32 [h, w] on the device; 1 inside, (dist/radius)^2 towards the border."""
    return torch.from_numpy(feather_mask_np(w, h, ratio)).to(host.device())


def custom_bbox_rect(x: float, y: float, w: float, h: float, canvas_w: int, canvas_h: int) -> Optional[Tuple[int, int, int, int]]:
    """Relative UI rectangle -> latent (x, y, w, h) (abstractdiffusion.py:206-215); None if the row is skipped."""
    out = (ctypes.c_int32 * 4)()
    if _cabi.check(_cabi.lib.td_custom_bbox_rect(float(x), float(y), float(w), float(h), int(canvas_w), int(canvas_h), out)) == 0:
        return None
    return int(out[0]), int(out[1]), int(out[2]), int(out[3])


class CustomBBox(BBox):
    """Region-control bbox (utils.py:84-99): a BBox plus its prompts, layer type, feather mask and seed."""

    __slots__ = ("prompt", "neg_prompt", "blend_mode", "feather_ratio", "seed", "feather_mask", "cond",
                 "extra_network_data", "uncond")

    def __init__(self, x: int, y: int, w: int, h: int, prompt: str, neg_prompt: str, blend_mode: str,
                 feather_radio: float, seed: int):
        super().__init__(x, y, w, h)
        self.prompt = prompt
        self.neg_prompt = neg_prompt
        self.blend_mode = BlendMode(blend_mode)
        self.feather_ratio = max(min(feather_radio, 1.0), 0.0)
        self.seed = seed
        self.feather_mask = feather_mask(self.w, self.h, self.feather_ratio) if self.blend_mode == BlendMode.FOREGROUND else None
        self.cond = None                  # MulticondLearnedConditioning of (global prompt, region prompt)
        self.extra_network_data = None    # parsed <lora:...> tags of the region prompt
        self.uncond = None                # learned conditioning of (global negative, region negative)


class Prompt:
    """utils.py:100-112."""

    @staticmethod
    def apply_styles(prompts: List[str], styles=None) -> List[str]:
        if not styles:
            return prompts
        shared = host.get_shared()
        return [shared.prompt_styles.apply_styles_to_prompt(p, styles) for p in prompts]

    @staticmethod
    def append_prompt(prompts: List[str], prompt: str = "") -> List[str]:
        if not prompt:
            return prompts
        return [f"{p}, {prompt}" for p in prompts]


class Condition:
    """CLIP conditioning through the host application's prompt parser (utils.py:114-147).  Outside the WebUI
    there is no text encoder: every method raises RuntimeError naming the missing module."""

    @staticmethod
    def _module(name: str):
        m = host.a1111_module(name)
        if m is None:
            raise RuntimeError(f"region prompts need the WebUI's modules.{name}; it is not importable here")
        return m

    @staticmethod
    def get_custom_cond(prompts: List[str], prompt: str, steps: int, styles=None):
        prompt = Prompt.apply_styles([prompt], styles)[0]
        _, extra_network_data = Condition._module("extra_networks").parse_prompts([prompt])
        prompts = Prompt.apply_styles(Prompt.append_prompt(prompts, prompt), styles)
        return Condition.get_cond(prompts, steps), extra_network_data

    @staticmethod
    def get_cond(prompts: List[str], steps: int):
        prompts, _ = Condition._module("extra_networks").parse_prompts(prompts)
        return Condition._module("prompt_parser").get_multicond_learned_conditioning(host.get_shared().sd_model, prompts, steps)

    @staticmethod
    def get_uncond(neg_prompts: List[str], steps: int, styles=None):
        neg_prompts = Prompt.apply_styles(neg_prompts, styles)
        return Condition._module("prompt_parser").get_learned_conditioning(host.get_shared().sd_model, neg_prompts, steps)

    @staticmethod
    def reconstruct_cond(cond, step: int) -> torch.Tensor:
        _, tensor = Condition._module("prompt_parser").reconstruct_multicond_batch(cond, step)
        return tensor

    @staticmethod
    def reconstruct_uncond(uncond, step: int) -> torch.Tensor:
        return Condition._module("prompt_parser").reconstruct_cond_batch(uncond, step)


def get_retouch_mask(img_input: np.ndarray, kernel_size: int) -> np.ndarray:
    """Where a self-guided box filter changes a grayscale image (utils.py:216-247): the high-frequency map noise
    inversion uses to decide where fresh noise is injected.  uint8-quantised, in [0, 1], float32 [H, W].

    Guided filter with guide == input: a = var / (var + 0.01), b = mean - a * mean over kernel x kernel boxes
    (OpenCV's normalised box blur, reflect-101 borders), out = mean_box(a) * I + mean_box(b)... the reference resizes
    a and b to the input size instead of blurring them, which at its fixed step of 1 is the identity."""
    import cv2
    img = img_input.astype(np.float32) / 255.0
    box = (int(round(kernel_size)), int(round(kernel_size)))
    mean_i = cv2.blur(img, box)
    mean_ii = cv2.blur(img * img, box)
    var_i = mean_ii - mean_i * mean_i
    a = var_i / (var_i + 0.01)                 # cov(I, p) == var(I) because p is I
    b = mean_i - a * mean_i
    gf = a * img + b
    gf -= img
    gf *= 255
    gf = gf.astype(np.uint8).clip(0, 255)
    return gf.astype(np.float32) / 255.0
