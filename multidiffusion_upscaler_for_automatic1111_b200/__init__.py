"""H100-native tiled-diffusion + tiled-VAE hot path behind the reference's API.

Drop-in for `pkuliyi2015/multidiffusion-upscaler-for-automatic1111`'s tile-method
delegates (`MultiDiffusion`, `MixtureOfDiffusers`) and `tilevae.VAEHook`: Python
host classes with the reference's names and arguments, calling hand-written
sm_90a CUDA kernels through the C-ABI in `include/td_b200.h`.

Importing this package loads `libtd_b200.so`; if it is missing the import fails
(there is no CPU / PyTorch fallback).
"""
from . import _cabi  # noqa: F401  (loads the shared library or raises)
from .tile_methods import AbstractDiffusion, DemoFusion, MixtureOfDiffusers, MultiDiffusion, SpotDiffusion
from .tile_utils.utils import BBox, Method, gaussian_weights, split_bboxes, splitable
from .tilevae import GroupNormParam, VAEHook

__all__ = ["AbstractDiffusion", "MultiDiffusion", "MixtureOfDiffusers", "DemoFusion", "SpotDiffusion", "VAEHook", "GroupNormParam", "BBox", "Method", "split_bboxes",
           "splitable", "gaussian_weights"]
