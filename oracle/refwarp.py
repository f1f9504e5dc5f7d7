"""ctypes binding of oracle/_ref/libref_warp.so: the REFERENCE's own CUDA warp kernel
(stnbdhw/BilinearSamplerBDHW.cu:48-109), extracted and compiled for sm_90a by oracle/Makefile behind
oracle/ref_warp/harness.cu.  TEST INFRASTRUCTURE ONLY: the pin of the warp oracle (tests/) and the "kernel to beat"
that bench.py times beside the product's warp.  Needs a CUDA device."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libref_warp.so")
_LIB = None


def available() -> bool:
    return os.path.exists(SO)


def lib():
    global _LIB
    if _LIB is None:
        if not available():
            raise FileNotFoundError(f"{SO} missing: run `make -C oracle refwarp` where /root/reference exists")
        _LIB = C.CDLL(SO)
        _LIB.ref_warp_bdhw_update_output.restype = C.c_int
    return _LIB


def _i4(v):
    return (C.c_int * 4)(*[int(x) for x in v])


def warp(img, grid, out=None):
    """img [B,C,Hin,Win], grid [B,2,Hout,Wout] CUDA fp32 tensors (any strides) -> out [B,C,Hout,Wout], launched on
    torch's current stream with the reference launcher's grid/block (BilinearSamplerBDHW.cu:119-120)."""
    import torch

    assert img.is_cuda and grid.is_cuda and img.dtype == torch.float32 and grid.dtype == torch.float32
    B, Cc, _, _ = img.shape
    Ho, Wo = grid.shape[-2:]
    if out is None:
        out = torch.empty((B, Cc, Ho, Wo), device=img.device, dtype=torch.float32)
    rc = lib().ref_warp_bdhw_update_output(C.c_void_p(img.data_ptr()), _i4(img.shape), _i4(img.stride()),
                                           C.c_void_p(grid.data_ptr()), _i4(grid.stride()), C.c_void_p(out.data_ptr()),
                                           _i4(out.stride()), Ho, Wo, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise RuntimeError(f"reference warp kernel launch failed: cudaError {rc}")
    return out
