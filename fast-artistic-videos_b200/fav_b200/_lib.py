"""ctypes loader for libfav_b200.so (the C ABI declared in include/fav.h).

There is NO Python / CPU fallback: if the shared library is missing, import fails loudly; if no CUDA
device is present every compute call raises FavError (FAV_ERR_NO_DEVICE).
"""
from __future__ import annotations

import ctypes as C
import os

_PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG_DIR, "libfav_b200.so")

FAV_OK = 0
FAV_ERR_INVALID = 1
FAV_ERR_CUDA = 2
FAV_ERR_NOT_IMPLEMENTED = 3
FAV_ERR_IO = 4
FAV_ERR_UNSUPPORTED = 5
FAV_ERR_NO_DEVICE = 6

BORDER_PER_TAP = 0
BORDER_PAD_PIXEL = 1


class FavError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"libfav_b200 status {status}: {message}")
        self.status = status
        self.message = message


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "or fast-artistic-videos_b200/build.sh (nvcc, sm_90a). There is no CPU fallback."
    )

lib = C.CDLL(LIB_PATH)

_i64p = C.POINTER(C.c_int64)
_fp = C.c_void_p  # device pointers are passed as integers

# every symbol include/fav.h declares (tests/test_abi.py checks this list against the header)
SIGNATURES = {
    "fav_last_error": (C.c_char_p, []),
    "fav_version": (C.c_int, []),
    "fav_launch_count": (C.c_uint64, []),
    "fav_device_count": (C.c_int, []),
    "fav_bilinear_sampler_bdhw_update_output": (C.c_int, [_fp, _i64p, _i64p, _fp, _i64p, _i64p, _fp, _i64p, C.c_int, _fp]),
    "fav_bilinear_sampler_bdhw_update_grad_input": (C.c_int, []),
    "fav_bilinear_sampler_bdhw_update_grad_input_only_grid": (C.c_int, []),
    "fav_warp_image": (C.c_int, [_fp, C.c_int, C.c_int, C.c_int, _fp, C.c_int, C.c_int, _fp, C.c_int, _fp]),
    "fav_min_filter": (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_vgg_preprocess": (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_vgg_deprocess": (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_temporal_input": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_temporal_stage": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_first_frame_input": (C.c_int, [_fp, _fp, _fp, C.c_int, C.c_int, _fp]),
    "fav_temporal_mse": (C.c_int, [_fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp, _fp]),
    "fav_consistency_check": (C.c_int, [_fp, _fp, _fp, C.c_float, _fp, _fp, C.c_int, C.c_int, _fp]),
    "fav_compute_corners_workspace": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "fav_compute_corners": (C.c_int, [_fp, C.c_int, C.c_int, C.c_int, C.c_float, _fp, _fp, _fp, _fp]),
    "fav_median_filter": (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    "fav_vr_blend_sides": (C.c_int, [_fp, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int), _fp, _fp, _fp, _fp,
                                     C.c_int, _fp]),
    "fav_flo_read_header": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fav_flo_read": (C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.c_int]),
    "fav_pnm_read_header": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fav_pnm_read_f32": (C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.c_float]),
    "fav_bytes_to_planes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "fav_planes_to_png_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "fav_png_write": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "fav_pnm_read_u8": (C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fav_flo_read_raw": (C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fav_net_create": (C.c_int, [C.c_char_p, C.c_char_p, C.c_float, C.c_int, C.POINTER(C.c_void_p)]),
    "fav_net_destroy": (None, [C.c_void_p]),
    "fav_net_num_params": (C.c_int, [C.c_void_p]),
    "fav_net_param_info": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, _i64p, _i64p]),
    "fav_net_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "fav_net_finalize": (C.c_int, [C.c_void_p]),
    "fav_net_set_conv_impl": (C.c_int, [C.c_void_p, C.c_int]),
    "fav_net_forward": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, _fp, _fp]),
    "fav_net_profile": (C.c_int, [C.c_void_p, _fp, C.c_int, C.c_int, _fp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_float),
                                  C.POINTER(C.c_double), C.c_char_p, C.POINTER(C.c_int), _fp]),
    "fav_net_layer_output": (C.c_int, [C.c_void_p, C.c_int, _fp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), _fp]),
    "fav_debug_set_trace": (C.c_int, [_fp, C.c_size_t]),
    "fav_debug_trace_words": (C.c_size_t, []),
    "fav_run_image": (C.c_int, [C.c_void_p, _fp, _fp, C.c_int, C.c_int, _fp, _fp]),
    "fav_run_next_image": (C.c_int, [C.c_void_p, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp, _fp]),
    "fav_run_next_image_flows": (C.c_int, [C.c_void_p, _fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp]),
    "fav_session_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "fav_session_destroy": (None, [C.c_void_p]),
    "fav_session_set_image_model": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fav_session_run_image": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fav_session_run_next_image": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "fav_session_run_next_image_flows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "fav_session_frame_done": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int]),
    "fav_session_run_frame_bytes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "fav_video_pipeline_run": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_double)]),
    "fav_session_sync": (C.c_int, [C.c_void_p]),
    "fav_session_last_gpu_ms": (C.c_float, [C.c_void_p]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _f = getattr(lib, _name)  # AttributeError here == ABI drift: fail loudly
    _f.restype = _res
    _f.argtypes = _args


def last_error() -> str:
    return lib.fav_last_error().decode(errors="replace")


def check(status: int) -> None:
    if status != FAV_OK:
        raise FavError(status, last_error())


def i64x4(vals):
    return (C.c_int64 * 4)(*[int(v) for v in vals])


def dptr(t):
    """Device pointer of a CUDA torch tensor (or None)."""
    if t is None:
        return None
    assert t.is_cuda, "libfav_b200 operates on CUDA tensors only (no CPU fallback)"
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
