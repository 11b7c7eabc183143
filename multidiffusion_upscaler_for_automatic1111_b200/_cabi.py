"""ctypes binding of libtd_b200.so (the C-ABI declared in include/td_b200.h).

There is NO fallback: if the shared library is missing or does not export a
symbol the header declares, importing this module raises.  The product path
never routes through `oracle/` or a PyTorch re-implementation.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint32, c_void_p

import torch

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TD_B200_LIB") or os.path.join(_PKG_DIR, "libtd_b200.so")   # env override: tuning builds only

TD_OK = 0
TD_ERR_INVALID_ARG, TD_ERR_UNSUPPORTED, TD_ERR_CUDA, TD_ERR_CAPACITY = -1, -2, -3, -4
TD_F16, TD_BF16, TD_F32 = 0, 1, 2
TD_FLAG_FORCE_GENERIC = 1
TD_FLAG_NO_TMA = 2
TD_FLAG_TMA = 4
TD_FLAG_PIPELINE = 8
TD_FLAG_PEER_ASYNC = 16
TD_FLAG_NO_PDL = 32
TD_FLAG_ONE_PLANE = 64
TD_FLAG_STRIP = 128
TD_FLAG_DBG_NO_TILES = 0x100
TD_FLAG_ROWS = 0x400
TD_WRAP_X, TD_WRAP_Y = 1, 2
TD_MAX_GRID_DIM = 256
TD_MAX_BATCH_PTRS = 128
TD_MAX_PEERS = 16
TD_IPC_HANDLE_BYTES = 64
ABI_VERSION = 13

DTYPE_CODE = {torch.float16: TD_F16, torch.bfloat16: TD_BF16, torch.float32: TD_F32}


class TdError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"td_b200 error {status}: {message}")
        self.status = status


class TdGrid(ctypes.Structure):
    """struct td_grid (include/td_b200.h)."""
    _fields_ = [
        ("H", c_int32), ("W", c_int32),
        ("tile_h", c_int32), ("tile_w", c_int32),
        ("overlap", c_int32),
        ("rows", c_int32), ("cols", c_int32),
        ("num_tiles", c_int32), ("num_batches", c_int32), ("tile_bs", c_int32),
        ("wrap", c_int32),
        ("ys", c_int32 * TD_MAX_GRID_DIM),
        ("xs", c_int32 * TD_MAX_GRID_DIM),
    ]


TD_MAX_REGIONS = 32


class TdRegion(ctypes.Structure):
    """struct td_region (include/td_b200.h)."""
    _fields_ = [("x", c_int32), ("y", c_int32), ("w", c_int32), ("h", c_int32), ("mode", c_int32), ("out", c_void_p), ("aux", c_void_p)]


class TdPushRegion(ctypes.Structure):
    """struct td_push_region (include/td_b200.h)."""
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("planes", c_int32), ("rows", c_int32), ("row_bytes", c_int64),
                ("src_plane_bytes", c_int64), ("src_pitch_bytes", c_int64), ("dst_plane_bytes", c_int64), ("dst_pitch_bytes", c_int64)]


TD_MAX_PUSH_REGIONS = 8
TD_PUSH_CTAS = 32


class TdConvDesc(ctypes.Structure):
    """struct td_conv_desc (include/td_b200.h)."""
    _fields_ = [
        ("N", c_int32), ("H", c_int32), ("W", c_int32), ("Cin", c_int32), ("Cout", c_int32),
        ("kh", c_int32), ("kw", c_int32), ("stride", c_int32), ("pad_top", c_int32), ("pad_left", c_int32),
        ("OH", c_int32), ("OW", c_int32), ("dtype", c_int32), ("bias_per_row", c_int32),
        ("alpha", c_float),
        ("x_pitch", c_int64), ("w_pitch", c_int64), ("y_pitch", c_int64), ("res_pitch", c_int64),
        ("post_scale", c_void_p), ("post_shift", c_void_p), ("post_act", c_int32),
        ("y2", c_void_p), ("y2_pitch", c_int64),
    ]


# symbol -> (restype, argtypes); must list EVERY function td_b200.h declares
_SIGNATURES = {
    "td_last_error": (c_char_p, []),
    "td_abi_version": (c_int, []),
    "td_debug_launch_empty": (c_int, [c_int, c_int, c_void_p]),
    "td_split_bboxes": (c_int, [c_int, c_int, c_int, c_int, c_int, POINTER(c_int32), c_int, POINTER(c_int), POINTER(c_int)]),
    "td_splitable": (c_int, [c_int, c_int, c_int, c_int, c_int]),
    "td_gaussian_weights": (c_int, [c_int, c_int, POINTER(c_float)]),
    "td_feather_mask": (c_int, [c_int, c_int, c_double, POINTER(c_float)]),
    "td_custom_bbox_rect": (c_int, [c_double, c_double, c_double, c_double, c_int, c_int, POINTER(c_int32)]),
    "td_grid_init": (c_int, [POINTER(TdGrid), c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "td_grid_weights": (c_int, [POINTER(TdGrid), POINTER(c_float), POINTER(c_float)]),
    "td_rescale_factor": (c_int, [POINTER(c_float), POINTER(c_float), c_int64]),
    "td_scatter_tiles": (c_int, [POINTER(TdGrid), c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_uint32, c_void_p]),
    "td_blend_multidiffusion": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
    "td_debug_check_fast_div": (c_int, [c_int, c_int, c_void_p, c_void_p]),
    "td_vae_best_tile_size": (c_int, [c_int, c_int]),
    "td_vae_split_tiles": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int32), POINTER(c_int32), c_int]),
    "td_nchw_to_nhwc_wrap": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, c_int64, c_int64,
                                     c_int, c_int, c_void_p]),
    "td_gn_stats_workspace_bytes": (c_int64, [c_int64, c_int64, c_int]),
    "td_gn_stats": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "td_gn_apply": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                            c_float, c_int, c_void_p]),
    "td_copy_region": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "td_resample_nearest": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "td_affine_clamp": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "td_dev_alloc": (c_int, [c_int64, POINTER(c_void_p)]),
    "td_dev_free": (c_int, [c_void_p]),
    "td_ipc_get_handle": (c_int, [c_void_p, c_void_p]),
    "td_ipc_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "td_ipc_close": (c_int, [c_void_p]),
    "td_peer_signal": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p, c_void_p]),
    "td_blend_multidiffusion_peer": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_uint32, c_void_p]),
    "td_blend_multidiffusion_rows": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                             c_uint32, c_void_p]),
    "td_blend_mixture_rows": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                      c_uint32, c_void_p]),
    "td_blend_multidiffusion_wrap_rows": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                                  c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                                  c_uint32, c_void_p]),
    "td_blend_mixture_wrap_rows": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                           c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                           c_uint32, c_void_p]),
    "td_peer_wait": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "td_push_regions": (c_int, [POINTER(TdPushRegion), c_int, POINTER(c_void_p), c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "td_region_composite": (c_int, [c_void_p, c_void_p, POINTER(TdRegion), c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "td_region_composite_rows": (c_int, [c_void_p, c_void_p, POINTER(TdRegion), c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                         c_int, c_int, c_void_p]),
    "td_dilated_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int32),
                                  POINTER(c_int32), POINTER(c_int32), c_int, c_int, c_void_p]),
    "td_demofusion_combine": (c_int, [c_void_p, POINTER(c_void_p), c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                      c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p]),
    "td_scatter_bboxes": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_void_p]),
    "td_blend_bboxes": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_void_p, c_void_p]),
    "td_demofusion_combine_offset": (c_int, [c_void_p, POINTER(c_void_p), c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int,
                                             c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p]),
    "td_depthwise_conv2d": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), c_int, c_int, c_void_p]),
    "td_depthwise_conv2d_wrap": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), c_int, c_int, c_int, c_void_p]),
    "td_scatter_bboxes_wrap": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_void_p]),
    "td_blend_bboxes_wrap": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "td_conv2d_nhwc": (c_int, [POINTER(TdConvDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "td_upconv2x_nhwc": (c_int, [POINTER(TdConvDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "td_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_int64, c_int64, c_int64, c_float, c_int,
                             c_void_p]),
    "td_nchw_to_nhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int, c_int, c_void_p]),
    "td_nhwc_to_nchw_region": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_int, c_int64, c_int64, c_int64, c_int64,
                                       c_int, c_void_p]),
    "td_upsample2x_nhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "td_gn_stats_nhwc_workspace_bytes": (c_int64, [c_int64, c_int, c_int]),
    "td_gn_stats_nhwc": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "td_gn_apply_nhwc": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int,
                                 c_void_p]),
    "td_softmax_rows": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_void_p]),
    "td_blend_mixture": (c_int, [POINTER(TdGrid), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int,
                                 c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
}


def _load() -> ctypes.CDLL:
    if not os.path.isfile(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found. Build it with `python -m multidiffusion_upscaler_for_automatic1111_b200.build` "
            "(needs nvcc). There is no CPU / PyTorch fallback for this path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError(f"{LIB_PATH} does not export `{name}` declared in include/td_b200.h") from e
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.td_abi_version() != ABI_VERSION:
        raise ImportError(f"ABI mismatch: library {lib.td_abi_version()} vs binding {ABI_VERSION}; rebuild")
    return lib


lib = _load()


def exported_symbols():
    return sorted(_SIGNATURES)


def check(status: int) -> int:
    """Raise TdError for a negative td_status; pass non-negative results through."""
    if status < 0:
        raise TdError(status, lib.td_last_error().decode("utf-8", "replace"))
    return status


def current_stream_ptr(device=None) -> c_void_p:
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return DTYPE_CODE[dtype]
    except KeyError:
        raise TypeError(f"unsupported dtype {dtype}; this path handles float16 / bfloat16 / float32") from None
