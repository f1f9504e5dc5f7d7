"""The activation arena on the CPU: the product's buffer planner (plan_arena, arena_plan.hpp) over the operands and steps of
the stylization net as build_plan lays them out (tests/emu/arena_emu.cu), at 720p, 4K and 8K, one frame and a batch of four.
No two operands that are live at the same time share a byte, every operand a step reads is written before it and still holds
its bytes, and the arena is smaller than the operands in buffers of their own."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

from fav_b200 import synth

EMU = os.path.join(ROOT, "tests", "emu")
DOUBLED = "c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3"
WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_arena.so")
    srcs = [os.path.join(EMU, f) for f in ("arena_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("arena_plan.hpp", "conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def plan_rows(arch, ptype, in_dim=7):
    """The net's layers in execution order as emu_arena_check reads them (see batch_emu.cu)."""
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


@pytest.mark.parametrize("shape", [(720, 1280), (2160, 3840), (4320, 7680)], ids=["720p", "4K", "8K"])
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("bn", [False, True], ids=["IN", "BN"])
@pytest.mark.parametrize("arch,ptype", [
    (synth.DEFAULT_ARCH, "reflect-start"),
    (synth.DEFAULT_ARCH, "zero"),
    (synth.PAPER_ARCH, "reflect-start"),
    (DOUBLED, "reflect-start"),
    (WIDE, "reflect-start"),
])
def test_arena_plan(emu, arch, ptype, bn, B, shape):
    H, W = shape
    rows = plan_rows(arch, ptype)
    R = synth.reflect_start_pad(synth.parse_arch(arch), ptype)
    flat = (C.c_int * (8 * len(rows)))(*[v for r in rows for v in r])
    out = (C.c_int64 * 4)()
    rc = emu.emu_arena_check(len(rows), flat, H + 2 * R, W + 2 * R, int(bn), B, out)
    assert rc == 0, emu.emu_last_error().decode()
    all_live, arena, nops, kept = list(out)
    print(f"{arch} {ptype} {'BN' if bn else 'IN'} B={B} {W}x{H}: operands all-live {all_live / 2**30:.2f} GiB, "
          f"arena {arena / 2**30:.2f} GiB ({nops - 1} operands, {kept} kept)")
    assert 0 < arena < all_live
    assert kept >= 1  # the input of the final layer
