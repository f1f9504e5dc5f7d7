"""Stacked sub-pixel phases on the CPU: the emulation of conv_tc_kernel running the stacked jobs of a stride-2 transposed
convolution (tests/emu/phase_stack_emu.cu, sharing the planner's plan_phase_stack / pack_phase_weights / stack_bias /
fill_conv_job and the kernel's stack_epi_addr) against a direct transposed convolution: patch staging, hi / lo weights packed
with zeros where a tap does not feed a phase, each phase's output placement and statistics channel.  The norm-on-load producers
of a stacked job stage the bytes the bulk copies stage from the in_apply'd operand."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_phase_stack.so")
    srcs = [os.path.join(EMU, f) for f in ("phase_stack_emu.cu", "nl_geom_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def plan(emu, cin, cout, k, H, W):
    out = (C.c_int * 9)()
    assert emu.emu_stack_plan(cin, cout, k, H, W, out) == 0, emu.emu_last_error().decode()
    jobs = [dict(zip(("Npad", "nstack", "taps", "b_resident"), out[1 + 4 * s:5 + 4 * s])) for s in range(min(out[0], 2))]
    return out[0], jobs


def test_planner_decisions_for_the_720p_layers(emu):
    n, jobs = plan(emu, 64, 32, 3, 360, 640)  # u32: all four phases, N = 4 x 32, taps (dy, dx) in {0, 1}^2
    assert n == 1 and jobs[0] == dict(Npad=128, nstack=4, taps=4, b_resident=jobs[0]["b_resident"])
    n, jobs = plan(emu, 128, 64, 3, 180, 320)  # u64: the two column phases of each row phase, N = 2 x 64
    assert n == 2 and [(j["Npad"], j["nstack"], j["taps"]) for j in jobs] == [(128, 2, 2), (128, 2, 4)]
    assert plan(emu, 256, 128, 3, 90, 160)[0] == 0  # u128 of the doubled arch: 2 x 128 > 128, one job per phase
    assert plan(emu, 64, 72, 3, 20, 30)[0] == 0
    n, jobs = plan(emu, 32, 48, 3, 20, 30)
    assert n == 2 and all(j["Npad"] == 96 for j in jobs)
    n, jobs = plan(emu, 32, 8, 3, 20, 30)
    assert n == 1 and jobs[0]["Npad"] == 32


CASES = [  # cin, cout, k, H, W
    (128, 64, 3, 5, 320),    # u64 at the 720p width: two jobs of N = 128, three tiles per row
    (64, 32, 3, 4, 640),     # u32 at the 720p width: one job of N = 128, five tiles per row
    (128, 64, 3, 3, 200),    # a width that is not a multiple of 128
    (64, 32, 3, 3, 129),     # a 1-pixel last tile
    (32, 8, 3, 4, 70),       # Cout 8: four phases, N = 32
    (32, 48, 3, 4, 70),      # Cout 48: two jobs, N = 96
    (8, 16, 3, 4, 70),       # from 8 channels (tap pairing), four phases, N = 64
    (32, 16, 5, 5, 70),      # f5s2: taps -1..1
    (64, 32, 7, 5, 70),      # f7s2: taps -1..2
    (64, 32, 9, 5, 70),      # f9s2: taps -2..2
]


@pytest.mark.parametrize("case", CASES)
def test_stacked_jobs_match_direct_transposed_conv(emu, case):
    me, mr, se = C.c_double(), C.c_double(), C.c_double()
    rc = emu.emu_stack_check(*case, 7, C.byref(me), C.byref(mr), C.byref(se))
    assert rc == 0, emu.emu_last_error().decode()
    assert me.value <= 2e-6 * max(mr.value, 1.0), (me.value, mr.value)  # ~2^-21: hi*hi + lo*hi + hi*lo
    assert se.value <= 1e-4, se.value  # statistics: each stored value in its phase's channel (a wrong channel is O(1) off)


def test_cout_72_is_not_stacked(emu):
    me, mr, se = C.c_double(), C.c_double(), C.c_double()
    assert emu.emu_stack_check(64, 72, 3, 4, 70, 7, C.byref(me), C.byref(mr), C.byref(se)) == 2
    assert "not stacked" in emu.emu_last_error().decode()


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("case", [(64, 32, 3, 6, 640), (64, 32, 3, 5, 129), (128, 64, 3, 4, 200), (32, 16, 5, 4, 70)])
def test_stacked_norm_on_load_stages_the_in_apply_operand(emu, case, B):
    info = (C.c_int * 3)()
    rc = emu.emu_stack_nl_check(*case, B, 99 + B, info)
    assert rc == 0, emu.emu_last_error().decode()
    assert info[0] >= 1 and info[1] > 0
