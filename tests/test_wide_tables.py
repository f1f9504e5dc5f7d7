"""Stylization nets wider than 128 channels per layer, on the CPU: every convolution with Cout > 128 runs as one conv_tc_kernel
job per 128-channel N block (and per sub-pixel phase).  The CPU emulation of those jobs (tests/emu/style_nblock_emu.cu,
emu_style_nblock_check) is driven by the product's planner, weight slicing and statistics placement and compared with a
direct convolution; nets the planner cannot run are refused by fav_net_finalize, by layer name, before any device work."""
import ctypes as C
import os
import subprocess

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_style_nblock.so")
    srcs = [os.path.join(EMU, f) for f in ("style_nblock_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


@pytest.mark.parametrize("case,jobs", [
    # cin, cout, k, stride, pad, transposed, adj, H, W
    ((7, 144, 9, 1, 4, 0, 0, 4, 140), 2),      # first conv c9s1-144: tap pairing, 2 N blocks, the last one 16 wide
    ((128, 256, 3, 2, 1, 0, 0, 6, 262), 2),    # d256: parity-split input, 2 N blocks, two tiles per output row
    ((256, 256, 3, 1, 0, 0, 0, 5, 134), 2),    # R256 residual conv, 'reflect-start' (pad 0)
    ((256, 256, 3, 1, 1, 0, 0, 3, 130), 2),    # R256 residual conv, 'zero' padding (pad 1)
    ((256, 192, 3, 2, 1, 1, 1, 3, 66), 8),     # u192: 4 sub-pixel phases x 2 N blocks (128 + 64)
    ((256, 160, 5, 2, 2, 1, 1, 3, 66), 8),     # f5s2-160: phases with 9/6/6/4 taps x 2 N blocks (128 + 32)
    ((64, 144, 3, 1, 1, 1, 0, 3, 130), 2),     # f3s1-144: stride-1 full convolution (flipped filter), 2 N blocks
    ((208, 384, 3, 2, 1, 0, 0, 4, 70), 3),     # d384 from 208 channels (CbG 2): three N blocks
])
def test_emulated_style_nblock_jobs_match_direct_conv(emu, case, jobs):
    me, mr, se, nj = C.c_double(), C.c_double(), C.c_double(), C.c_int()
    rc = emu.emu_style_nblock_check(*case, 5, C.byref(me), C.byref(mr), C.byref(se), C.byref(nj))
    assert rc == 0, emu.emu_last_error().decode()
    assert nj.value == jobs
    assert me.value <= 2e-6 * max(mr.value, 1.0), (me.value, mr.value)  # ~2^-21: hi*hi + lo*hi + hi*lo
    assert se.value <= 2e-6, se.value  # each block's statistics land in its own channels' slots


def _finalize_error(arch, padding_type="reflect-start", in_dim=7, norm="instance"):
    from fav_b200 import _lib, models_video, synth

    net = models_video.StyleNet(arch, padding_type=padding_type, in_dim=in_dim, norm=norm)
    try:
        net.load_state(synth.make_weights(arch, "candy", in_dim, norm=norm))
    except _lib.FavError as e:
        return e
    return None


@pytest.mark.parametrize("arch,layer", [
    ("c9s1-32,d64,d576,R576,u64,u32,c9s1-3", "l3.c1"),  # 3x3 conv from 576 channels: 18 channel groups > 16 K groups
    ("c9s1-32,d64,R64,u256,c9s1-3", "l4"),              # final c9s1-3 from 256 channels: the x-fold plan needs 24 K groups
    ("c9s1-32,d64,d200,R200,u64,u32,c9s1-3", "l3.c1"),  # Cin 200: not a multiple of 16
])
def test_unplannable_wide_nets_are_refused_at_finalize(arch, layer):
    """Refused in fav_net_finalize with FAV_ERR_UNSUPPORTED and the layer's name, before any device work (so also here,
    without a GPU), never at the first forward."""
    from fav_b200 import _lib

    e = _finalize_error(arch)
    assert e is not None and e.status == _lib.FAV_ERR_UNSUPPORTED, e
    assert f"conv {layer}:" in str(e), str(e)


@pytest.mark.parametrize("arch,ptype", [
    ("c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3", "reflect-start"),
    ("c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3", "zero"),
    ("c9s1-64,d128,d256,R256,R256,U2,c3s1-128,U2,c9s1-3", "reflect-start"),
    ("c9s1-144,d208,d384,R384,u208,u128,c9s1-3", "reflect-start"),
    ("c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3", "reflect-start"),
])
def test_wide_nets_pass_planning(arch, ptype):
    """The wide archs of the GPU tests plan: finalize gets past the planner (without a GPU it then stops at the device)."""
    import torch

    from fav_b200 import _lib

    e = _finalize_error(arch, ptype)
    if torch.cuda.is_available():
        assert e is None, e
    else:
        assert e is not None and e.status == _lib.FAV_ERR_NO_DEVICE, e
