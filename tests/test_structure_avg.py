"""The exact parallel CMatrix::avg (exact_avg.cuh) on the CPU: tests/emu/avg_emu.cu runs the kernels' records, estimate and
combine walk on the host with the helpers the kernels use, and must give the bits of the plain sequential fp32 loop
a = fl(a + x_k), avg = fl(a / n) (CMatrix.h:1245-1251) on every input, including negative values, cancellation, ties,
absorbed elements, subnormals, NaN and Inf."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_avg.so")
    srcs = [os.path.join(EMU, "avg_emu.cu"), os.path.join(ROOT, "fast-artistic-videos_b200", "csrc", "exact_avg.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_avg_seq.restype = C.c_float
    lib.emu_avg_seq.argtypes = [C.c_void_p, C.c_int64]
    lib.emu_avg_exact.restype = C.c_float
    lib.emu_avg_exact.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def run(emu, x):
    x = np.ascontiguousarray(x, np.float32)
    stats = np.zeros(3, np.int64)
    got = np.float32(emu.emu_avg_exact(x.ctypes.data, x.size, stats.ctypes.data))
    ref = np.float32(emu.emu_avg_seq(x.ctypes.data, x.size))
    assert got.tobytes() == ref.tobytes(), (x.size, got, ref)
    return stats


def test_sequential_loop_is_the_reference(emu):
    # the reference is the loop the oracle's orc_avg runs; its sum in numpy's own order would differ
    x = np.random.default_rng(0).uniform(size=100_003).astype(np.float32)
    a = np.float32(0)
    for v in x[:5000]:
        a = np.float32(a + v)
    assert np.float32(emu.emu_avg_seq(x[:5000].ctypes.data, 5000)) == np.float32(a / np.float32(5000))


SIZES = {"1": 1, "2": 2, "sub-1": 255, "sub": 256, "sub+1": 257, "chunk-1": 8191, "chunk": 8192, "chunk+1": 8193,
         "720p": 1280 * 720, "1080p": 1920 * 1080, "2048sq": 2048 * 2048, "4k": 3840 * 2160}


@pytest.mark.parametrize("size", list(SIZES))
def test_uniform(emu, size):
    n = SIZES[size]
    stats = run(emu, np.random.default_rng(n).uniform(size=n))
    if n >= 1280 * 720:  # the walk takes the jumps: most of the data is never summed element by element
        assert stats[2] * 256 < n // 8, stats


@pytest.mark.parametrize("shape", [(720, 1280), (1080, 1920), (2048, 2048), (2160, 3840)])
def test_corner_maps(emu, shape):
    """pyoracle.compute_corners of synthetic frames: normalize's `else if` quirk can leave early elements below the minimum."""
    from fav_b200 import synth
    from oracle import pyoracle

    H, W = shape
    img = np.clip(np.rint(synth.make_frame(H, W, 2) * 255.0), 0, 255).astype(np.float32)
    img[:, :, : W // 3] = 128.0
    run(emu, pyoracle.compute_corners(img).ravel())


def test_corner_map_with_negatives(emu):
    from oracle import pyoracle

    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, size=(3, 200, 300)).astype(np.float32)
    img[:, :20, :20] = 90.0  # flat top-left: the first corners are strict prefix maxima below the scan's minimum
    c = pyoracle.compute_corners(img).ravel()
    assert (c < 0).any()
    run(emu, c)
    run(emu, np.tile(c, 20))


def test_ties_at_large_sums(emu):
    """x = 2^-8 once |a| > 2^16: every step is an exact tie between two fp32 neighbours (parity decides)."""
    for n in (300_000, 2_000_000):
        x = np.full(n, 2.0 ** -8, np.float32)
        x[:70_000] = 1.0
        assert run(emu, x)[0] > 0  # the ties are resolved inside jumped chunks, not only by FADDs
    x = np.full(1_000_000, 0.5, np.float32)  # ties at 2^23 and above
    x[:20] = 2.0 ** 22
    run(emu, x)
    x = np.random.default_rng(1).choice(np.float32([0.125, 0.375, 0.0625, 1.0]), size=1_500_000)
    run(emu, x)


def test_mixed_signs_cancel_across_binades(emu):
    rng = np.random.default_rng(2)
    n = 1_000_000
    run(emu, rng.normal(0, 1, size=n))
    ramp = np.concatenate([np.ones(300_000), -np.ones(300_000), np.full(300_000, 0.7), -np.full(350_000, 1.3)])
    run(emu, ramp + rng.uniform(-1e-3, 1e-3, size=ramp.size))
    run(emu, -rng.uniform(size=n))


def test_special_values(emu):
    n = 100_000
    run(emu, np.zeros(n))
    run(emu, -np.zeros(n))
    run(emu, np.full(n, 0.3))
    run(emu, np.full(n, 1.0))
    x = np.full(n, 1e-4, np.float32)
    x[0] = 3e7  # one huge value, then small ones absorbed entirely
    run(emu, x)
    x[5000] = -3e7
    run(emu, x)
    run(emu, np.full(n, 1e-40, np.float32))  # subnormals
    x = np.random.default_rng(4).uniform(size=n).astype(np.float32)
    x[::7] = 1e-42
    run(emu, x)
    for bad in (np.inf, -np.inf, np.nan):
        y = x.copy()
        y[70_000] = bad
        run(emu, y)
    y = x.copy()
    y[10] = 3e38
    y[11] = 3e38  # overflow to Inf in the middle of the chain
    run(emu, y)
