"""Emulation of the stylization net's single-pass fp16 mode (fav_net_set_precision "fp16") on NetOracle's operand_round hook.
TEST INFRASTRUCTURE ONLY.  Every convolution multiplies fp16(x) (round to nearest: what the hi plane of the operand holds)
with the fp16 hi halves the product packs (fp16(w 2^e) 2^-e, from tests/emu/fp16_mode_emu.cu: weight_half and the conv's
power-of-two prescale), accumulating in fp64; everything else is NetOracle's fp64."""
import ctypes as C
import os
import subprocess

import numpy as np
import torch
import torch.nn.functional as F

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_LIB = None


def emu_lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(EMU, "libfav_emu_fp16_mode.so")
        if not os.path.exists(so):
            subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                                   "-Wno-deprecated-gpu-targets", "-o", so, os.path.join(EMU, "fp16_mode_emu.cu")])
        _LIB = C.CDLL(so)
        _LIB.emu_last_error.restype = C.c_char_p
    return _LIB


def packed_hi_weights(w: np.ndarray, transposed: bool) -> np.ndarray:
    """fp16 hi halves of a conv's weights as the product packs them, in weight units (float64, same shape)."""
    w = np.ascontiguousarray(w, dtype=np.float32)
    a, b, k = w.shape[0], w.shape[1], w.shape[2]
    cin, cout = (a, b) if transposed else (b, a)
    out = np.empty(w.size, np.float64)
    e = C.c_int()
    rc = emu_lib().emu_fp16_weight_hi(cin, cout, k, 1, 0, int(transposed), 0, w.ctypes.data_as(C.c_void_p),
                                      out.ctypes.data_as(C.c_void_p), C.byref(e))
    assert rc == 0, emu_lib().emu_last_error().decode()
    return out.reshape(w.shape)


class Fp16Round:
    """operand_round hook: round=False gives back the plain fp64 convolution (the emulator's identity check)."""

    def __init__(self, round_operands: bool = True):
        self.round = round_operands
        self._cache = {}

    def __call__(self, x, wt, b, kw, transposed):
        if self.round:
            x = x.to(torch.float16).to(x.dtype)
            key = (wt.data_ptr(), tuple(wt.shape))
            if key not in self._cache:
                self._cache[key] = torch.from_numpy(packed_hi_weights(wt.cpu().numpy(), transposed)).to(wt.dtype).to(wt.device)
            wt = self._cache[key]
        return F.conv_transpose2d(x, wt, b, **kw) if transposed else F.conv2d(x, wt, b, **kw)


def fp16_oracle(**kw):
    from oracle import net_oracle
    return net_oracle.NetOracle(dtype=torch.float64, operand_round=Fp16Round(True), **kw)
