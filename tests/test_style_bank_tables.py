"""Style banks on the CPU: the emulation of how conv_tc_kernel's batched instances pick each image's style (tests/emu/
style_bank_emu.cu, sharing the kernel's style_at and the product's planner and slot chooser) over the plans of the GPU tests'
archs.  Every tile of every CTA reads the weight chunks, bias, 2^-w_exp, norm-on-load table and operand-epilogue scale of its
own image's style; the producers announce the bytes they copy, for the fp16 pair and the single pass; a banked job streams its
weights (a CTA's tiles cross styles, so no weight stays resident)."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

from fav_b200 import synth

EMU = os.path.join(ROOT, "tests", "emu")
PAPER = synth.PAPER_ARCH
DOUBLED = "c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3"
H100_SMS = 132


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_style_bank.so")
    srcs = [os.path.join(EMU, f) for f in ("style_bank_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh", "conv_tc.cu")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def plan_rows(arch, ptype, in_dim=7):
    """The net's layers in execution order as emu_style_bank_check reads them (batch_emu.cu's format)."""
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


def check(emu, arch, ptype, bn, styles, H, W, single=0, allow_resident=0):
    rows = plan_rows(arch, ptype)
    R = synth.reflect_start_pad(synth.parse_arch(arch), ptype)
    flat = (C.c_int * (8 * len(rows)))(*[v for r in rows for v in r])
    st = (C.c_int * len(styles))(*styles)
    info = (C.c_int * 5)()
    rc = emu.emu_style_bank_check(len(rows), flat, H + 2 * R, W + 2 * R, int(bn), len(styles), st, max(styles) + 1, H100_SMS,
                                  single, allow_resident, info)
    assert rc == 0, emu.emu_last_error().decode()
    return dict(jobs=info[0], nl=info[1], opnd=info[2], switches=info[3], resident=info[4])


STYLES = {
    2: {"distinct": [1, 0], "repeat": [1, 1]},
    5: {"distinct": [4, 2, 0, 3, 1], "repeat": [2, 0, 2, 2, 0]},
    9: {"distinct": [8, 3, 5, 0, 7, 1, 6, 2, 4], "repeat": [2, 0, 1, 2, 2, 0, 1, 1, 0]},
}


@pytest.mark.parametrize("shape", [(64, 96), (720, 1280)])
@pytest.mark.parametrize("B", [2, 5, 9])
@pytest.mark.parametrize("kind", ["distinct", "repeat"])
@pytest.mark.parametrize("arch,ptype,bn", [
    (synth.DEFAULT_ARCH, "reflect-start", False),
    (PAPER, "reflect-start", False),
    (DOUBLED, "reflect-start", False),
    (synth.DEFAULT_ARCH, "reflect-start", True),
    (synth.DEFAULT_ARCH, "zero", False),
])
def test_every_tile_reads_its_images_style(emu, arch, ptype, bn, kind, B, shape):
    H, W = shape
    styles = STYLES[B][kind]
    for single in (0, 1):
        r = check(emu, arch, ptype, bn, styles, H, W, single)
        assert r["jobs"] > 0 and r["resident"] == 0, r
        assert (r["opnd"] > 0) == bn
        assert bn or r["nl"] > 0
        if len(set(styles)) > 1 and H == 720:
            assert r["switches"] > 0, r  # some CTA's tiles cross from one style to another


def test_resident_weights_would_serve_the_wrong_style(emu):
    """The check has teeth: kept resident (as they are for a net with one style), the small layers' weights of a CTA's first tile
    serve its later tiles, which at 256x256 belong to an image of another style."""
    with pytest.raises(AssertionError, match="outside its style.s packed weights|weight chunk of another style"):
        check(emu, synth.DEFAULT_ARCH, "reflect-start", False, [0, 1], 256, 256, allow_resident=1)
    r = check(emu, synth.DEFAULT_ARCH, "reflect-start", False, [0, 0], 256, 256, allow_resident=1)
    assert r["resident"] > 0


def test_a_single_style_batch_switches_nothing(emu):
    r = check(emu, synth.DEFAULT_ARCH, "reflect-start", False, [0, 0, 0], 256, 256)
    assert r["switches"] == 0 and r["resident"] == 0


def test_add_style_refuses_unfinalized_nets():
    """Both nets must be finalized (fav_net_finalize); checked before any device work, so without a GPU as well."""
    import ctypes

    from fav_b200 import _lib, models_video

    a, b = models_video.StyleNet(synth.DEFAULT_ARCH), models_video.StyleNet(synth.DEFAULT_ARCH)
    idx = ctypes.c_int(-1)
    assert _lib.lib.fav_net_add_style(a._h, b._h, ctypes.byref(idx)) == _lib.FAV_ERR_INVALID
    assert "finalized" in _lib.last_error() and idx.value == -1
    assert a.num_styles == 1
    # an assignment names styles the net holds: a fresh net has style 0 only
    assert _lib.lib.fav_net_set_batch_styles(a._h, (ctypes.c_int * 2)(0, 1), 2) == _lib.FAV_ERR_INVALID
    assert "holds 1" in _lib.last_error()
    assert _lib.lib.fav_net_set_batch_styles(a._h, (ctypes.c_int * 2)(0, 0), 2) == _lib.FAV_OK
    assert _lib.lib.fav_net_set_batch_styles(a._h, None, 0) == _lib.FAV_OK
