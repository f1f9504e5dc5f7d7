"""Norm-on-load on the CPU: the emulation of conv_tc_kernel's norm-on-load producers (tests/emu/nl_geom_emu.cu, sharing the
kernel's nl_raw_row / nl_raw_col and the planner's set_norm_on_load / nl_geometry_ok) against the stage the bulk copies fill
from the operand in_apply writes.  Every consumer geometry the planner fuses -- stride-2 parity-split convs, the sub-pixel phase
jobs of transposed convs, the x-fold final conv, plain and tap-paired convs, the second conv of every block -- at 720p, at the
tile-edge sizes of the GPU arch-geometry table, single image and batched: the staged operand bits are the ones the unfused
plan stages, so the fused net computes exactly what the unfused one does."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

from fav_b200 import synth
from test_batch_tables import plan_rows
from test_gpu_arch_geometry import ROWS

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_nl_geom.so")
    srcs = [os.path.join(EMU, f) for f in ("nl_geom_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def check(emu, arch, ptype, B, H, W, in_dim=7):
    rows = plan_rows(arch, ptype, in_dim)
    R = synth.reflect_start_pad(synth.parse_arch(arch, in_dim), ptype)
    flat = (C.c_int * (8 * len(rows)))(*[v for r in rows for v in r])
    info = (C.c_int * 4)()
    rc = emu.emu_nl_geometry_check(len(rows), flat, H + 2 * R, W + 2 * R, B, 1234 + B, info)
    assert rc == 0, emu.emu_last_error().decode()
    return list(info)


# default arch: l0 -> d64 and d64 -> d128 (parity split), u64 -> u32 (four phase jobs), u32 -> the x-fold final conv, and
# the second conv of each of the five residual blocks
DEFAULT_FUSED = 4 + 5
# paper arch: the two stride-2 convs and the five residual blocks (its upsamplings normalise in up_apply)
PAPER_FUSED = 2 + 5


@pytest.mark.parametrize("ptype", ["reflect-start", "zero"])
def test_default_arch_at_720p(emu, ptype):
    fused, jobs, cells, past = check(emu, synth.DEFAULT_ARCH, ptype, 1, 720, 1280)
    assert fused == DEFAULT_FUSED
    assert jobs == 2 + 4 + 1 + 5
    assert cells > 0


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("shape", [(64, 96), (48, 508), (16, 16)])
@pytest.mark.parametrize("arch,ptype,fused", [
    (synth.DEFAULT_ARCH, "reflect-start", DEFAULT_FUSED),
    (synth.DEFAULT_ARCH, "zero", DEFAULT_FUSED),
    (synth.PAPER_ARCH, "reflect-start", PAPER_FUSED),
])
def test_released_archs(emu, arch, ptype, fused, shape, B):
    H, W = shape
    assert check(emu, arch, ptype, B, H, W)[0] == fused


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("name", sorted(ROWS))
def test_arch_geometry_rows(emu, name, B):
    arch, ptype, in_dim, H, W = ROWS[name]
    fused, jobs, _, _ = check(emu, arch, ptype, B, H, W, in_dim)
    assert fused >= 1 and jobs >= fused
