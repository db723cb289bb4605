"""ctypes binding of libpww_b200.so (the C ABI in include/pww_b200.h).

There is no fallback: if the library is missing or a call returns a non-zero status this module
raises.  `PWW_B200_LIB` overrides the library path.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PWW_B200_LIB", os.path.join(_HERE, "libpww_b200.so"))

PWW_STAT_MAX, PWW_STAT_STD = 0, 1
PWW_DTYPE_F32, PWW_DTYPE_F16, PWW_DTYPE_BF16 = 0, 1, 4     # 2 and 3 are unassigned (unsupported, as before bf16)

EXPORTS = (
    "pww_version", "pww_status_str", "pww_last_cuda_error", "pww_device_supported",
    "pww_xattn_workspace_bytes", "pww_xattn_stats_f16", "pww_xattn_fwd_f16", "pww_attn_fwd_f16",
    "pww_xattn_fused_workspace_bytes", "pww_xattn_fused_f16",
    "pww_xattn_stats_multi_f16", "pww_xattn_fwd_multi_f16", "pww_xattn_fused_multi_f16",
    "pww_groupnorm_workspace_bytes", "pww_groupnorm_nhwc_f16", "pww_geglu_f16", "pww_add_layernorm_f16",
    "pww_sampler_input", "pww_sampler_update",
    "pww_xattn_stats_bf16", "pww_xattn_fwd_bf16", "pww_xattn_fused_bf16",
    "pww_xattn_stats_multi_bf16", "pww_xattn_fwd_multi_bf16", "pww_xattn_fused_multi_bf16",
    "pww_attn_fwd_bf16", "pww_groupnorm_nhwc_bf16", "pww_geglu_bf16", "pww_add_layernorm_bf16",
    "pww_control_inject_f16", "pww_control_inject_bf16",
    "pww_control_combine_f16", "pww_control_combine_bf16",
    "pww_resnet_residual_f16", "pww_resnet_residual_bf16",
    "pww_xattn_fused_rec_f16", "pww_xattn_fused_rec_bf16",
    "pww_adapter_residual_f16", "pww_adapter_residual_bf16",
    "pww_sampler_update_rescale", "pww_sampler_update_masked",
    "pww_window_input", "pww_window_update",
    "pww_xattn_fused_region_f16", "pww_xattn_fused_region_bf16",
    "pww_xattn_fused_region_multi_f16", "pww_xattn_fused_region_multi_bf16",
    "pww_xattn_fused_region_rows_f16", "pww_xattn_fused_region_rows_bf16",
    "pww_xattn_fused_region_rows_multi_f16", "pww_xattn_fused_region_rows_multi_bf16",
)


class NativeError(RuntimeError):
    pass


_lib: Optional[ctypes.CDLL] = None
launch_count = 0          # kernels launched through this binding (bench.py reports it as gpu_launches)


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            f"{LIB_PATH} not found: build it with `python -m paint_with_words_sd_b200.csrc.build` "
            "(there is no CPU / PyTorch fallback for the attention path)")
    L = ctypes.CDLL(LIB_PATH)
    c_i, c_i64, c_vp, c_f, c_sz = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_float, ctypes.c_size_t
    L.pww_version.restype = c_i
    L.pww_status_str.restype = ctypes.c_char_p
    L.pww_status_str.argtypes = [c_i]
    L.pww_last_cuda_error.restype = ctypes.c_char_p
    L.pww_device_supported.restype = c_i
    L.pww_xattn_workspace_bytes.restype = c_sz
    L.pww_xattn_workspace_bytes.argtypes = [c_i] * 5
    L.pww_xattn_stats_f16.restype = c_i
    L.pww_xattn_stats_f16.argtypes = [c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64, c_i, c_vp,
                                      c_vp, c_vp, c_sz, c_vp]
    L.pww_xattn_fwd_f16.restype = c_i
    L.pww_xattn_fwd_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64,
                                    c_i64, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_f, c_vp]
    L.pww_xattn_fused_workspace_bytes.restype = c_sz
    L.pww_xattn_fused_workspace_bytes.argtypes = []
    L.pww_xattn_fused_f16.restype = c_i
    L.pww_xattn_fused_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64,
                                      c_i64, c_i64, c_vp, c_i64, c_i, c_vp, c_vp, c_i, c_vp, c_f, c_vp, c_vp, c_sz, c_vp]
    # per-image twins: `stat` is an int32 [B] device array instead of an int, `g_sigma` holds B values
    L.pww_xattn_stats_multi_f16.restype = c_i
    L.pww_xattn_stats_multi_f16.argtypes = [c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp,
                                            c_vp, c_vp, c_sz, c_vp]
    L.pww_xattn_fwd_multi_f16.restype = c_i
    L.pww_xattn_fwd_multi_f16.argtypes = list(L.pww_xattn_fwd_f16.argtypes)
    L.pww_xattn_fused_multi_f16.restype = c_i
    L.pww_xattn_fused_multi_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64,
                                            c_i64, c_i64, c_vp, c_i64, c_i, c_vp, c_vp, c_vp, c_vp, c_f, c_vp, c_vp, c_sz,
                                            c_vp]
    # the _multi arguments, then ridx, rec_index, rec_acc (device pointers) and rec_batch_stride (elements)
    L.pww_xattn_fused_rec_f16.restype = c_i
    L.pww_xattn_fused_rec_f16.argtypes = list(L.pww_xattn_fused_multi_f16.argtypes) + [c_vp, c_vp, c_vp, c_i64]
    # region prompts: the fused (or _multi) arguments, then region_weights (device pointer) and its batch stride
    L.pww_xattn_fused_region_f16.restype = c_i
    L.pww_xattn_fused_region_f16.argtypes = list(L.pww_xattn_fused_f16.argtypes) + [c_vp, c_i64]
    L.pww_xattn_fused_region_multi_f16.restype = c_i
    L.pww_xattn_fused_region_multi_f16.argtypes = list(L.pww_xattn_fused_multi_f16.argtypes) + [c_vp, c_i64]
    # negative region prompts: the region arguments, then region_index and stat_chunks (device pointers or NULL)
    L.pww_xattn_fused_region_rows_f16.restype = c_i
    L.pww_xattn_fused_region_rows_f16.argtypes = list(L.pww_xattn_fused_region_f16.argtypes) + [c_vp, c_vp]
    L.pww_xattn_fused_region_rows_multi_f16.restype = c_i
    L.pww_xattn_fused_region_rows_multi_f16.argtypes = list(L.pww_xattn_fused_region_multi_f16.argtypes) + [c_vp, c_vp]
    L.pww_attn_fwd_f16.restype = c_i
    L.pww_attn_fwd_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64, c_f, c_vp]
    L.pww_groupnorm_workspace_bytes.restype = c_sz
    L.pww_groupnorm_workspace_bytes.argtypes = [c_i, c_i, c_i]
    L.pww_groupnorm_nhwc_f16.restype = c_i
    L.pww_groupnorm_nhwc_f16.argtypes = [c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_f, c_i, c_vp, c_sz, c_vp]
    L.pww_geglu_f16.restype = c_i
    L.pww_geglu_f16.argtypes = [c_vp, c_vp, c_i64, c_i, c_vp]
    L.pww_add_layernorm_f16.restype = c_i
    L.pww_add_layernorm_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i, c_f, c_vp]
    L.pww_resnet_residual_f16.restype = c_i
    L.pww_resnet_residual_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i64, c_i, c_vp]
    # a, b, bias (or NULL), feat (or NULL), out, rows, pixels, C, feat_rows, stream
    L.pww_adapter_residual_f16.restype = c_i
    L.pww_adapter_residual_f16.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, c_i, c_i64, c_i, c_i, c_vp]
    # n, dst[n], res[n], elems_per_image[n] (host arrays), rows, scales (device [n, rows] fp32 or NULL), stream
    L.pww_control_inject_f16.restype = c_i
    L.pww_control_inject_f16.argtypes = [c_i, ctypes.POINTER(c_vp), ctypes.POINTER(c_vp), ctypes.POINTER(c_i64), c_i,
                                         c_vp, c_vp]
    # units, n, out[n], res[units * n], elems_per_image[n] (host arrays), rows, scales (device [units, n, rows]), stream
    L.pww_control_combine_f16.restype = c_i
    L.pww_control_combine_f16.argtypes = [c_i, c_i, ctypes.POINTER(c_vp), ctypes.POINTER(c_vp), ctypes.POINTER(c_i64),
                                          c_i, c_vp, c_vp]
    # every _bf16 entry point takes its _f16 twin's arguments
    for name in EXPORTS:
        if name.endswith("_bf16"):
            twin = getattr(L, name[:-len("_bf16")] + "_f16")
            fn = getattr(L, name)
            fn.restype, fn.argtypes = twin.restype, list(twin.argtypes)
    L.pww_sampler_input.restype = c_i
    L.pww_sampler_input.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i, c_i, c_i, c_i, c_i, c_vp]
    L.pww_sampler_update.restype = c_i
    L.pww_sampler_update.argtypes = [c_vp, c_i, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_i, c_vp, c_vp, c_vp, c_vp,
                                     c_i, c_i, c_i, c_vp]
    # pww_sampler_update's arguments with rescale [m] and stats_out [m, 3] (or NULL) after `form`
    L.pww_sampler_update_rescale.restype = c_i
    L.pww_sampler_update_rescale.argtypes = L.pww_sampler_update.argtypes[:13] + [c_vp, c_vp] + \
        L.pww_sampler_update.argtypes[13:]
    # pww_sampler_update_rescale's arguments up to stats_out, then init_latents, init_noise, mask and sigma_next
    L.pww_sampler_update_masked.restype = c_i
    L.pww_sampler_update_masked.argtypes = L.pww_sampler_update_rescale.argtypes[:15] + [c_vp] * 4 + \
        L.pww_sampler_update.argtypes[13:]
    # latents, scale, row_starts, n_rows, col_starts, n_cols, first_view, n_views, window, out, out_dtype, h, w, stream
    L.pww_window_input.restype = c_i
    L.pww_window_input.argtypes = [c_vp, c_vp, c_vp, c_i, c_vp, c_i, c_i, c_i, c_i, c_vp, c_i, c_i, c_i, c_vp]
    # eps[n_chunks] (host array), n_chunks, views_per_chunk, eps_dtype, 4 strides, row_starts, n_rows, col_starts,
    # n_cols, window, then pww_sampler_update's latents .. form, height, width, stream
    L.pww_window_update.restype = c_i
    L.pww_window_update.argtypes = [ctypes.POINTER(c_vp), c_i, c_i, c_i, c_i64, c_i64, c_i64, c_i64, c_vp, c_i, c_vp,
                                    c_i, c_i] + L.pww_sampler_update.argtypes[6:13] + [c_i, c_i, c_vp]
    _lib = L
    return L


def entry(name: str, dtype):
    """The C entry point `name` (without its type suffix) for element type `dtype`: `_bf16` for torch.bfloat16, else
    `_f16`."""
    return getattr(lib(), name + ("_bf16" if dtype == torch.bfloat16 else "_f16"))


def check(status: int, what: str) -> None:
    if status != 0:
        L = lib()
        msg = L.pww_status_str(status).decode()
        if status == -3:
            msg += ": " + L.pww_last_cuda_error().decode()
        raise NativeError(f"{what} failed: {msg} (status {status})")
