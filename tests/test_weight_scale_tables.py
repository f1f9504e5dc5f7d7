"""The power-of-two weight prescale of every tensor-core convolution (set_weight_prescale / weight_half, conv_plan.hpp), on the
CPU through tests/emu/conv_emu.cu.  The tensor cores multiply with fp16 pairs w 2^e = hi + lo.  Without the 2^e, a weight below
2^-3 leaves lo in the fp16 subnormals and an absolute error of up to 2^-25 whatever its size: a conv with max |w| = 2^-40 would
multiply with zeros.  For every packing path (N blocks, sub-pixel phases, stacked phases, x-fold, tap pairing, stride 2, the
row-fold image and the phase-fold job) and max |w| from 2^-40 to 2^3:
- each packed pair times 2^-e gives back its weight to 2^-21 of itself, or of the fp16 pair's floor 2^-4 (2^-4-e in weight
  units), and that floor is at most 2^-19 of max |w|;
- a conv with max |w| in [2^-6, 2^15) keeps e = 0 (its packing bit for bit as without the scale); below, max |w| 2^e lies in
  [2^14, 2^15), clear of the fp16 maximum, and the floor drops to 2^-39 of max |w|;
- every job of a conv runs with the same e."""
import ctypes as C

import pytest

from test_conv_tables import emu  # noqa: F401  (module fixture: builds and loads libfav_emu.so)

# name: cin, cout, k, stride, pad, transposed, adj, raw_out, path (0: the jobs the nets pack, 1: row-fold image, 2: phase-fold)
CASES = {
    "first-conv-tap-pairing": (7, 32, 9, 1, 4, 0, 0, 1, 0),
    "stride2-parity-split": (32, 64, 3, 2, 1, 0, 0, 1, 0),
    "residual-generic": (128, 128, 3, 1, 0, 0, 0, 1, 0),
    "nblocks-cout-320": (64, 320, 3, 1, 1, 0, 0, 1, 0),           # three N blocks (128 + 128 + 64)
    "nblocks-loss-cin512": (512, 256, 3, 1, 1, 0, 0, 1, 0),       # VGG conv4: 16 channel groups, two N blocks
    "u64-stacked-pairs": (128, 64, 3, 2, 1, 1, 1, 1, 0),          # two stacked jobs of two sub-pixel phases
    "u32-stacked-four": (64, 32, 3, 2, 1, 1, 1, 1, 0),            # one stacked job of four phases
    "f3s2-192-phase-nblocks": (256, 192, 3, 2, 1, 1, 1, 1, 0),     # four phases x two N blocks (transposed slices)
    "f5s2-phases": (32, 80, 5, 2, 2, 1, 1, 1, 0),                 # 2 Cout > 128: one job per phase (9/6/6/4 taps)
    "xfold-final": (32, 3, 9, 1, 4, 0, 0, 0, 0),
    "rowfold-tap-pairing": (7, 32, 9, 1, 4, 0, 0, 1, 1),
    "rowfold-xfold": (32, 3, 9, 1, 4, 0, 0, 0, 1),
    "phase-fold": (64, 32, 3, 2, 1, 1, 1, 1, 2),
}
EXPONENTS = sorted(set(range(-40, 4, 3)) | {-6, -5, 3})  # max |w| = 0.999 2^L: L = -5 is the smallest unscaled conv


def check(emu, case, wscale, seed=1):
    out, e = (C.c_double * 5)(), C.c_int()
    rc = emu.emu_weight_scale_check(*case, C.c_double(wscale), seed, out, C.byref(e))
    assert rc == 0, emu.emu_last_error().decode()
    return dict(worst=out[0], top=out[1], jobs=int(out[2]), exps=int(out[3]), unseen=int(out[4]), e=e.value)


@pytest.mark.parametrize("name", list(CASES))
def test_packed_pairs_reproduce_weights_at_every_scale(emu, name):
    case = CASES[name]
    for L in EXPONENTS:
        r = check(emu, case, 2.0 ** L)
        where = f"{name}, max |w| ~ 2^{L}: {r}"
        assert r["worst"] <= 1.0, where                  # |(hi + lo) 2^-e - w| <= 2^-21 max(|w|, 2^-4-e)
        assert r["exps"] == 1, where                     # one exponent for every job of the conv
        assert r["unseen"] == 0, where                   # every weight is packed by some job
        if L >= -5:                                      # max |w| in [2^-6, 2^15): unscaled
            assert r["e"] == 0 and 2.0 ** -6 <= r["top"] < 2.0 ** 15, where
        else:                                            # max |w| 2^e in [2^14, 2^15): hi stays below 65504
            assert r["e"] == 14 - (L - 1) and 2.0 ** 14 <= r["top"] < 2.0 ** 15, where
        assert 2.0 ** -25 / r["top"] <= 2.0 ** -19, where  # the floor, relative to max |w|


@pytest.mark.parametrize("name", ["residual-generic", "u32-stacked-four", "nblocks-cout-320", "xfold-final", "phase-fold"])
def test_all_zero_conv_gets_exponent_zero(emu, name):
    r = check(emu, CASES[name], 0.0)
    assert r["e"] == 0 and r["exps"] == 1 and r["worst"] == 0.0, r


def test_job_counts(emu):
    """The enumeration covers what it names: N blocks x phases, stacked jobs, single row-fold / phase-fold jobs."""
    jobs = {n: check(emu, CASES[n], 0.1)["jobs"] for n in CASES}
    assert jobs["nblocks-cout-320"] == 3 and jobs["nblocks-loss-cin512"] == 2
    assert jobs["u64-stacked-pairs"] == 4 + 2 and jobs["u32-stacked-four"] == 4 + 1  # per-phase jobs (batch-normalized nets) too
    assert jobs["f3s2-192-phase-nblocks"] == 8 and jobs["f5s2-phases"] == 4
    assert jobs["rowfold-xfold"] == jobs["phase-fold"] == 1
