"""Batches on the CPU: the emulation of how conv_tc_kernel walks a batch of images (tests/emu/batch_emu.cu, sharing the kernel's
tile decode tile_at and opnd_epi_addr) over the plans of the GPU tests' archs.  Every (image, tile) runs exactly once, every
address of image b stays inside image b's region of its tensor, and each CTA's tiles of one image are the tiles some CTA runs
when that image runs alone -- the reason a batched image is bit-identical to the image run alone (DESIGN.md 4.1)."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

from fav_b200 import synth

EMU = os.path.join(ROOT, "tests", "emu")
PAPER = synth.PAPER_ARCH
WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"
H100_SMS = 132


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_batch.so")
    srcs = [os.path.join(EMU, f) for f in ("batch_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def plan_rows(arch, ptype, in_dim=7):
    """The net's layers in execution order as emu_batch_check reads them (see batch_emu.cu)."""
    rows = []
    bp = 1 if ptype == "zero" else 0
    for s in synth.parse_arch(arch, in_dim):
        if s["kind"] == "conv":
            rows.append([0, s["cin"], s["cout"], s["k"], s["stride"], s["pad"], 0, 0])
        elif s["kind"] == "fullconv":
            rows.append([0, s["cin"], s["cout"], s["k"], s["stride"], s["pad"], 1, s["adj"]])
        elif s["kind"] == "up":
            rows.append([1, s["cin"], s["cout"], 0, s["scale"], 0, 0, 0])
        else:
            rows.append([2, s["cin"], s["cout"], 3, 1, bp, 0, 0])
            rows.append([3 if s["skip"] else 4, s["cout"], s["cout"], 3, 1, bp, 0, 0])
    return rows


def check(emu, arch, ptype, bn, B, H, W):
    rows = plan_rows(arch, ptype)
    R = synth.reflect_start_pad(synth.parse_arch(arch), ptype)
    flat = (C.c_int * (8 * len(rows)))(*[v for r in rows for v in r])
    info = (C.c_int * 4)()
    rc = emu.emu_batch_check(len(rows), flat, H + 2 * R, W + 2 * R, H, W, int(bn), B, H100_SMS, info)
    assert rc == 0, emu.emu_last_error().decode()
    return list(info)


@pytest.mark.parametrize("shape", [(64, 96), (48, 508), (16, 16)])
@pytest.mark.parametrize("B", [1, 2, 3, 5])
@pytest.mark.parametrize("arch,ptype,bn", [
    (synth.DEFAULT_ARCH, "reflect-start", False),
    (synth.DEFAULT_ARCH, "zero", False),
    (PAPER, "reflect-start", False),
    (synth.DEFAULT_ARCH, "reflect-start", True),
    (WIDE, "reflect-start", False),
])
def test_batched_tiles_and_addresses(emu, arch, ptype, bn, B, shape):
    H, W = shape
    jobs, nl, opnd, wider = check(emu, arch, ptype, bn, B, H, W)
    assert jobs > 0
    assert (opnd > 0) == bn
    assert nl > 0 or bn or "R" not in arch and "C" not in arch
    if B == 1:
        assert wider == 0


def test_batch_grid_crosses_a_wave_only_for_the_batch(emu):
    """256x256: the residual convs have 64..82 tiles (fewer than the 132 SMs); two images need more CTAs than one."""
    _, _, _, wider = check(emu, synth.DEFAULT_ARCH, "reflect-start", False, 2, 256, 256)
    assert wider > 0
