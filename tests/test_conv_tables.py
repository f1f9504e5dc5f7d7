"""CPU emulation of the wgmma kernel's addressing (tests/emu/conv_emu.cu) against a direct convolution, for every
layer shape of the supported archs plus edge shapes: validates K-step tables, patch segments, parity-split input,
sub-pixel phases of the transposed convolution, weight packing and the fp16 hi/lo split (3-MMA scheme)."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu.so")
    src = os.path.join(EMU, "conv_emu.cu")
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


CASES = [  # cin, cout, k, stride, pad, transposed, adj, H, W
    (7, 32, 9, 1, 4, 0, 0, 10, 140),     # l0  c9s1-32 (Cin 7 -> 8, tap pairing)
    (32, 64, 3, 2, 1, 0, 0, 12, 268),    # l1  d64 (parity-split input)
    (64, 128, 3, 2, 1, 0, 0, 8, 260),    # l2  d128
    (128, 128, 3, 1, 0, 0, 0, 6, 134),   # residual convs
    (128, 64, 3, 2, 1, 1, 1, 5, 70),     # u64 (4 sub-pixel phases)
    (64, 32, 3, 2, 1, 1, 1, 5, 130),     # u32
    (32, 3, 9, 1, 4, 0, 0, 10, 132),     # last c9s1-3 (Cout 3 -> 16, row groups)
    (128, 64, 3, 1, 1, 0, 0, 5, 130),    # c3s1-64 of the paper arch
    (3, 32, 9, 1, 4, 0, 0, 9, 20),       # image model first layer, frame narrower than one tile
    (128, 128, 3, 1, 0, 0, 0, 3, 3),     # 1x1 output
    (32, 3, 9, 1, 4, 0, 0, 19, 250),     # final conv: R = 8 row-fold, partial last unit, 3 x-fold tiles (120-px stride)
    (7, 32, 9, 1, 4, 0, 0, 13, 300),     # conv1: R = 4 row-fold + K-split, partial last unit, 3 tiles
    (32, 64, 3, 2, 1, 0, 0, 14, 260),    # d64, K-split over 18 steps, odd tile remainder
    (128, 128, 3, 1, 0, 0, 0, 7, 320),   # residual conv: odd row count (last two-row unit half empty), 318-px rows
    (128, 64, 3, 2, 1, 1, 1, 4, 140),    # u64 phase-fold (N = 256, single issuer), two tiles
    (64, 32, 3, 2, 1, 1, 1, 3, 129),     # u32 phase-fold + K-split, one-pixel second tile
    (64, 3, 9, 1, 4, 0, 0, 11, 140),     # paper-arch final conv (64 channels): x-fold without row-fold
    (64, 32, 3, 1, 1, 1, 0, 6, 140),     # f3s1-32: stride-1 full convolution = convolution with the flipped filter
    (32, 16, 5, 2, 2, 1, 1, 5, 70),      # f5s2-16: four sub-pixel phases with 9/6/6/4 taps, tap offsets -1..1
    (64, 64, 3, 1, 1, 0, 0, 7, 150),     # residual conv of the 'zero' padding type (pad 1, 64 channels: conv_tc path)
    (16, 3, 9, 1, 4, 0, 0, 6, 130),      # final c9s1-3 from 16 channels: x-fold with CbG 2
    (32, 3, 5, 1, 2, 0, 0, 6, 260),      # final c5s1-3: x-fold with N = 5 x 3 -> 16, 124-px tile stride
    (8, 3, 9, 1, 4, 0, 0, 6, 140),       # final conv from 8 channels: tap pairing, plain final epilogue
    (32, 3, 3, 1, 1, 0, 0, 5, 129),      # final c3s1-3: generic plan, plain final epilogue
    (32, 8, 3, 2, 1, 1, 1, 4, 70),       # u8: Cout 8 in an N = 16 instance
]


@pytest.mark.parametrize("case", CASES)
def test_emulated_kernel_addressing_matches_direct_conv(emu, case):
    me, mr, sm, nm = C.c_double(), C.c_double(), C.c_int(), C.c_int()
    rc = emu.emu_conv_check(*case, 1, C.byref(me), C.byref(mr), C.byref(sm), C.byref(nm))
    assert rc == 0, emu.emu_last_error().decode()
    assert me.value <= 2e-6 * max(mr.value, 1.0), (me.value, mr.value)  # ~2^-21: hi*hi + lo*hi + hi*lo
    assert sm.value <= 227 * 1024


def plan(emu, *case):
    out = (C.c_int * 10)()
    assert emu.emu_plan_info(*case, out) == 0, emu.emu_last_error().decode()
    return dict(zip(("mt", "ksplit", "pf", "rf_R", "xfold_kw", "b_resident", "a_stages", "b_slots", "ntiles", "Npad"), out))


def test_planner_decisions_for_the_720p_layers(emu):
    """The plans conv_tc.cu runs (DESIGN.md section 4.1), at the sizes of the 720p frame: one output row per unit, one
    register accumulator of N <= 128 columns per warpgroup (no two-row units, K-split, row-fold or phase-fold)."""
    res = plan(emu, 128, 128, 3, 1, 0, 0, 0, 180, 320)
    assert res["mt"] == 1 and not res["ksplit"] and not res["b_resident"] and res["Npad"] == 128   # weights stream through the ring
    conv1 = plan(emu, 7, 32, 9, 1, 4, 0, 0, 800, 1360)
    assert conv1["rf_R"] == 0 and conv1["b_resident"] and conv1["Npad"] == 32
    final = plan(emu, 32, 3, 9, 1, 4, 0, 0, 720, 1280)
    assert final["rf_R"] == 0 and final["xfold_kw"] == 9 and final["Npad"] == 32        # x-fold: N = 9 x 3 -> 32
    u64 = plan(emu, 128, 64, 3, 2, 1, 1, 1, 180, 320)
    assert not u64["pf"] and u64["Npad"] == 64                                          # four sub-pixel phase jobs
    u32 = plan(emu, 64, 32, 3, 2, 1, 1, 1, 360, 640)
    assert not u32["pf"] and u32["Npad"] == 32 and u32["b_resident"]
    final64 = plan(emu, 64, 3, 9, 1, 4, 0, 0, 720, 1280)                                # paper arch: 64 input channels
    assert final64["rf_R"] == 0 and final64["xfold_kw"] == 9
    assert plan(emu, 32, 3, 5, 1, 2, 0, 0, 720, 1280)["xfold_kw"] == 5                  # c5s1-3: N = 15 -> 16
    for case in ((8, 3, 9, 1, 4, 0, 0, 720, 1280), (32, 3, 3, 1, 1, 0, 0, 720, 1280)):  # 8-channel input / 3x3: no x-fold
        assert plan(emu, *case)["xfold_kw"] == 0
    for case in ((32, 64, 3, 2, 1, 0, 0, 800, 1360), (64, 128, 3, 2, 1, 0, 0, 400, 680)):
        d = plan(emu, *case)
        assert d["mt"] == 1 and not d["ksplit"]
