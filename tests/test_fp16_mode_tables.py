"""The single-pass fp16 mode of conv_tc_kernel (ConvJob::single, fav_net_set_precision "fp16") on the CPU, through
tests/emu/fp16_mode_emu.cu: the planner's jobs for every plan kind (generic, stride-2 parity split, tap pairing, x-fold, stacked
sub-pixel phases, N blocks, a batch of images) run with the patch producer copying the hi plane only and the weight producer
the first half of each chunk, into stages and slots poisoned with NaNs.
- Each producer announces (expect-tx, the helpers the kernel calls) exactly the bytes it copies: a mismatch would hang the kernel.
- The hi prefix of every packed chunk holds exactly the hi steps the consumer reads: the emulated result equals a direct fp64
  convolution of fp16(x) with the packed hi weights to fp64 rounding, with no NaN read."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_fp16_mode.so")
    srcs = [os.path.join(EMU, f) for f in ("fp16_mode_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


# name: cin, cout, k, stride, pad, transposed, adj, H, W, mode (0: one job per phase / N block, 1: stacked phases), images
CASES = {
    "first-conv-tap-pairing": (7, 32, 9, 1, 4, 0, 0, 12, 140, 0, 1),
    "first-conv-from-3": (3, 32, 9, 1, 4, 0, 0, 10, 70, 0, 1),
    "stride2-parity-split": (32, 64, 3, 2, 1, 0, 0, 10, 270, 0, 1),
    "stride2-d128": (64, 128, 3, 2, 1, 0, 0, 8, 140, 0, 1),
    "residual-generic": (128, 128, 3, 1, 0, 0, 0, 8, 140, 0, 1),
    "residual-generic-batch3": (64, 64, 3, 1, 1, 0, 0, 6, 130, 0, 3),
    "nblocks-cout-320": (64, 320, 3, 1, 1, 0, 0, 5, 70, 0, 1),
    "u64-stacked-pairs": (128, 64, 3, 2, 1, 1, 1, 4, 140, 1, 1),
    "u32-stacked-four": (64, 32, 3, 2, 1, 1, 1, 4, 140, 1, 2),
    "f3s2-phases": (64, 32, 3, 2, 1, 1, 1, 4, 70, 0, 1),
    "f5s2-phases": (32, 80, 5, 2, 2, 1, 1, 4, 70, 0, 1),
    "xfold-final": (32, 3, 9, 1, 4, 0, 0, 6, 250, 0, 1),
    "xfold-final-batch2": (32, 3, 9, 1, 4, 0, 0, 5, 130, 0, 2),
}


def run(emu, case, seed=3):
    out = (C.c_double * 5)()
    rc = emu.emu_fp16_conv_check(*case, seed, out)
    assert rc == 0, emu.emu_last_error().decode()
    return dict(err=out[0], jobs=int(out[1]), a_tx=out[2], b_tx=out[3], nl_ok=int(out[4]))


@pytest.mark.parametrize("name", list(CASES))
def test_single_pass_producers_and_hi_prefix(emu, name):
    r = run(emu, CASES[name])
    assert r["jobs"] >= 1
    # fp64 sums of exact fp16 products: only the summation order differs from the direct convolution
    assert r["err"] < 1e-12, r


def test_announced_bytes_are_half_of_the_pair(emu):
    """One plane of each: the single-pass producers announce exactly half what the pair's producers announce, so a
    single-pass kernel never waits for bytes that no copy brings."""
    lib = emu
    for name, case in CASES.items():
        r = run(lib, case)
        cin, cout, k, stride, pad, tr, adj, H, W, mode, nimg = case
        if mode:
            continue
        detail = (C.c_int * 16)()
        assert lib.emu_plan_detail(cin, cout, k, stride, pad, tr, adj, H, W, detail) == 0, lib.emu_last_error().decode()
        chunk_bytes = detail[10]
        if cout <= 128 and not tr:  # one job: its weight chunk
            assert r["b_tx"] == chunk_bytes / 2, (name, r, chunk_bytes)


def test_norm_on_load_geometries_are_covered(emu):
    """The plain and parity-split patches are the ones norm-on-load fills (nl_geometry_ok): its producers write the hi plane
    only in this mode, the cells the bulk copies would fill (tests/emu/nl_geom_emu.cu checks that those cells agree)."""
    assert run(emu, CASES["residual-generic"])["nl_ok"] == 1
    assert run(emu, CASES["stride2-parity-split"])["nl_ok"] == 1


def test_weight_hi_halves_follow_the_prescale(emu):
    """emu_fp16_weight_hi (the oracle's weights) is fp16(w 2^e) 2^-e with the conv's power-of-two prescale: tiny weights keep
    11 significant bits instead of flushing to fp16 subnormals."""
    import numpy as np
    rng = np.random.default_rng(0)
    for scale in (1e-9, 1e-3, 0.1, 3.0):
        w = (rng.uniform(-1, 1, size=(16, 8, 3, 3)) * scale).astype(np.float32)
        out = np.empty(w.size, np.float64)
        e = C.c_int()
        assert emu.emu_fp16_weight_hi(8, 16, 3, 1, 1, 0, 0, w.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                                      C.byref(e)) == 0
        ref = np.ldexp(np.ldexp(w.astype(np.float64), e.value).astype(np.float16).astype(np.float64), -e.value)
        assert np.array_equal(out.reshape(w.shape), ref)
        assert np.abs(out.reshape(w.shape) - w).max() <= np.abs(w).max() * 2.0 ** -11
