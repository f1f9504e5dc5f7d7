"""-evaluate's perceptual loss network on the CPU side: utils.parse_layers, the Torch7 loss-network reader (trimming, cudnn.* and
SpatialConvolutionMM names, 2-D weights, ceil_mode, refusals), fav_percep_create's refusal of geometries the planner cannot
run, and the CPU emulation of the N-block convolution plan that runs
VGG-16's 256- and 512-channel layers (tests/emu/nblock_emu.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


def small_net(ceil_mode=True):
    """conv / ReLU / pool chain with the module types of loadcaffe's VGG, small channel counts"""
    rng = np.random.default_rng(5)
    conv = lambda ci, co: dict(type="conv", cin=ci, cout=co, k=3, stride=1, pad=1,
                               weight=rng.standard_normal((co, ci, 3, 3)).astype(np.float32), bias=rng.standard_normal(co).astype(np.float32))
    pool = dict(type="pool", kW=2, kH=2, dW=2, dH=2, padW=0, padH=0, ceil_mode=ceil_mode)
    return [conv(3, 16), dict(type="relu"), pool, conv(16, 32), dict(type="relu"), dict(pool), conv(32, 32), dict(type="relu")]


def test_parse_layers_semantics():
    from fav_b200 import percep

    assert percep.parse_layers("4,9,16,23", "1.0") == (["4", "9", "16", "23"], [1.0] * 4)  # one weight repeated (utils.lua:30-36)
    assert percep.parse_layers("16", "2.5") == (["16"], [2.5])
    assert percep.parse_layers("4,9", "1,3") == (["4", "9"], [1.0, 3.0])
    with pytest.raises(ValueError, match="size mismatch"):
        percep.parse_layers("4,9,16", "1,2")
    assert percep.layer_index("23") == 23
    from fav_b200 import _lib

    with pytest.raises(_lib.FavError) as e:
        percep.layer_index("2-1")  # nested layer strings (layer_utils.lua) address container children: refused
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "nested" in str(e.value)


@pytest.mark.parametrize("kind", ["nn", "cudnn", "mm"])
def test_loss_network_reader_round_trip_and_trim(tmp_path, kind):
    from fav_b200 import t7

    mods = small_net()
    p = str(tmp_path / "loss.t7")
    t7.write_loss_network(p, mods, classifier=True, cudnn=kind == "cudnn", conv_mm=kind == "mm")
    raw = t7.load(p)
    names = [raw["modules"][i].torch_type for i in sorted(raw["modules"])]
    assert names[-1] == "nn.SoftMax" and "nn.View" in names  # the classifier is in the file ...
    if kind == "mm":
        assert raw["modules"][1]["weight"].ndim == 2  # SpatialConvolutionMM stores [cout, cin*k*k]
    if kind == "cudnn":
        assert names[0] == "cudnn.SpatialConvolution"
    got = t7.load_loss_network(p, len(mods))  # ... and trimmed away: the deepest loss layer is the last ReLU
    assert [m["type"] for m in got] == [m["type"] for m in mods]
    for a, b in zip(got, mods):
        if a["type"] == "conv":
            assert a["weight"].shape == b["weight"].shape and np.array_equal(a["weight"], b["weight"])
            assert np.array_equal(a["bias"], b["bias"]) and (a["k"], a["stride"], a["pad"]) == (3, 1, 1)
        if a["type"] == "pool":
            assert a["ceil_mode"] is True and (a["kW"], a["dW"], a["padW"]) == (2, 2, 0)
    assert len(t7.load_loss_network(p, 4)) == 4  # trimmed after module 4


def test_loss_network_reader_refusals(tmp_path):
    from fav_b200 import _lib, t7

    mods = small_net()
    p = str(tmp_path / "loss.t7")
    t7.write_loss_network(p, mods, classifier=True)
    with pytest.raises(_lib.FavError) as e:  # a loss layer inside the classifier: nn.View (module 9) is before it
        t7.load_loss_network(p, len(mods) + 2)
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "module 9" in str(e.value) and "nn.View" in str(e.value)
    # a module type the GPU path does not run, before the deepest loss layer (e.g. a ResNet's batch norm)
    model = t7.load(p)
    model["modules"][2] = t7.T7Object("nn.SpatialBatchNormalization", {})
    with pytest.raises(_lib.FavError) as e:
        t7.loss_network_from_model(model, 4)
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "module 2" in str(e.value) and "SpatialBatchNormalization" in str(e.value)
    # a convolution geometry the tensor-core planner does not run (stride 3)
    model = t7.load(p)
    model["modules"][4]["dW"] = model["modules"][4]["dH"] = 3
    with pytest.raises(_lib.FavError) as e:
        t7.loss_network_from_model(model, 5)
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "module 4" in str(e.value)


def test_vgg16_shapes_and_default_layers():
    from fav_b200 import percep

    mods = percep.vgg16_modules(0)
    assert len(mods) == 31
    names = {4: "relu", 9: "relu", 16: "relu", 23: "relu", 5: "pool", 17: "pool"}
    for i, t in names.items():
        assert mods[i - 1]["type"] == t, i
    convs = [(m["cin"], m["cout"]) for m in mods if m["type"] == "conv"]
    assert convs[:10] == [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512)]


def _conv(cin, cout, k, stride=1, pad=None):
    return dict(type="conv", cin=cin, cout=cout, k=k, stride=stride, pad=k // 2 if pad is None else pad,
                weight=np.zeros((cout, cin, k, k), np.float32), bias=np.zeros(cout, np.float32))


@pytest.mark.parametrize("mods,module", [
    ([_conv(3, 128, 3), dict(type="relu"), _conv(128, 64, 7)], 3),  # 7 filter rows x 4 channel groups = 28 K groups > 16
    ([_conv(3, 16, 3), dict(type="relu"), _conv(16, 32, 5, stride=2)], 3),  # stride 2 is planned for k3 pad 1 only
    ([_conv(3, 24, 3), dict(type="relu"), _conv(24, 32, 3)], 3),  # Cin must be <= 8 or a multiple of 16
    ([_conv(3, 16, 3, stride=2)], 1),  # the parity-split operand needs Cin >= 16
    ([_conv(3, 8, 3), dict(type="relu"), _conv(8, 16, 3, stride=2)], 3),
])
def test_unplannable_convolutions_are_refused_at_create(mods, module):
    """A loss network the tensor-core planner cannot run fails in fav_percep_create, before any weights reach the GPU,
    with FAV_ERR_UNSUPPORTED and the module's index."""
    from fav_b200 import _lib, percep

    with pytest.raises(_lib.FavError) as e:
        percep.PerceptualCriterion(mods, [len(mods)], [1.0], [], [])
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and f"module {module}" in str(e.value), str(e.value)


@pytest.fixture(scope="module")
def nblock_emu():
    so = os.path.join(EMU, "libfav_emu_nblock.so")
    srcs = [os.path.join(EMU, f) for f in ("nblock_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


@pytest.mark.parametrize("case", [
    (512, 512, 3, 1, 2, 9),    # conv4_2 / conv4_3: 4 N blocks, Cin 512 = 16 K groups
    (256, 512, 3, 1, 3, 7),    # conv4_1: 4 N blocks, 8 K groups
    (128, 256, 3, 1, 2, 130),  # conv3_1: 2 N blocks, two tiles per row
    (64, 200, 3, 1, 2, 5),     # a partial last N block (72 channels, N = 80)
    # k >= 5, pad (k-1)/2 and Cout <= 4 (or a last N block that narrow): the stylization net's x-fold plan writes the final
    # tanh image, so a loss-network conv of that shape must get the generic plan
    (16, 3, 5, 2, 3, 9),
    (64, 130, 5, 2, 3, 9),     # last N block of 2 channels
    (32, 4, 7, 3, 2, 140),
])
def test_emulated_nblock_plan_matches_direct_conv(nblock_emu, case):
    cin, cout, k, pad, H, W = case
    me, mr, nj, ng = C.c_double(), C.c_double(), C.c_int(), C.c_int()
    rc = nblock_emu.emu_nblock_check(cin, cout, k, pad, H, W, 3, C.byref(me), C.byref(mr), C.byref(nj), C.byref(ng))
    assert rc == 0, nblock_emu.emu_last_error().decode()
    assert nj.value == (cout + 127) // 128
    assert ng.value <= 16 and (cin != 512 or ng.value == 16)
    assert me.value <= 2e-6 * max(mr.value, 1.0), (me.value, mr.value)
