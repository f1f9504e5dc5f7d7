"""Batch-normalized stylization nets (-use_instance_norm 0) on the CPU: .t7 round trips of SpatialBatchNormalization checkpoints,
the loader's refusals, the C ABI's BN parameter table and its refusal of invalid running statistics at fav_net_finalize, and
the CPU emulation of conv_tc_kernel's operand epilogue (tests/emu/opnd_epi_emu.cu) over the BN plans of the GPU tests' archs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

from fav_b200 import synth
from test_gpu_arch_geometry import BN_ROWS as GEOMETRY_BN_ROWS, ROWS as GEOMETRY_ROWS

EMU = os.path.join(ROOT, "tests", "emu")
PAPER = synth.PAPER_ARCH
WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"
# + the BN rows of the arch-geometry table: epilogues writing operands with padT 3 / 4 (c7s1 / c9s1 consumers) and tpad 2 - 4
# (f5s1 / f7s1 / f9s1 consumers)
ARCHS = [(synth.DEFAULT_ARCH, "reflect-start"), (synth.DEFAULT_ARCH, "zero"), (PAPER, "reflect-start"), (WIDE, "reflect-start")] + \
    [GEOMETRY_ROWS[name][:2] for name in GEOMETRY_BN_ROWS]


def _write_read(tmp_path, arch, w, **kw):
    from fav_b200 import t7

    p = str(tmp_path / "bn.t7")
    ptype = kw.get("padding_type", "reflect-start")
    t7.write_checkpoint(p, arch, w, reflect_pad=synth.reflect_start_pad(synth.parse_arch(arch), ptype), norm="batch", **kw)
    geo = {}
    got_arch, state, _, _ = t7.load_checkpoint(p, geo)
    return got_arch, state, geo


def _bn_weights(arch, seed=1):
    rng = np.random.default_rng(seed)
    w = synth.make_weights(arch, "candy", norm="batch")
    for k in w:
        if k.endswith(".running_mean") or k.endswith(".bias") and ".n" in k:
            w[k] = rng.normal(0, 1, w[k].shape).astype(np.float32)
        elif k.endswith(".running_var"):
            w[k] = rng.uniform(0.5, 2, w[k].shape).astype(np.float32)
    return w


@pytest.mark.parametrize("bn_class", ["nn.SpatialBatchNormalization", "cudnn.SpatialBatchNormalization"])
@pytest.mark.parametrize("arch,ptype", ARCHS[:3])  # write_checkpoint has no CX blocks
def test_bn_checkpoint_round_trip(tmp_path, bn_class, arch, ptype):
    w = _bn_weights(arch)
    got_arch, state, geo = _write_read(tmp_path, arch, w, padding_type=ptype, bn_class=bn_class)
    assert got_arch == arch and geo["norm"] == "batch" and geo["padding_type"] == ptype
    assert sorted(state) == sorted(w)
    for k in w:
        np.testing.assert_array_equal(state[k].reshape(-1), w[k].reshape(-1), err_msg=k)


def test_bn_checkpoint_without_affine_reads_weight_one_bias_zero(tmp_path):
    w = _bn_weights(synth.DEFAULT_ARCH)
    _, state, geo = _write_read(tmp_path, synth.DEFAULT_ARCH, w, affine=False)
    assert geo["norm"] == "batch"
    for k in w:
        if ".n" in k and k.endswith(".weight"):
            np.testing.assert_array_equal(state[k], np.ones_like(w[k]))
        elif ".n" in k and k.endswith(".bias"):
            np.testing.assert_array_equal(state[k], np.zeros_like(w[k]))
        else:
            np.testing.assert_array_equal(state[k].reshape(-1), w[k].reshape(-1), err_msg=k)


def test_instance_norm_checkpoint_reports_instance(tmp_path):
    from fav_b200 import t7

    p = str(tmp_path / "in.t7")
    t7.write_checkpoint(p, synth.DEFAULT_ARCH, synth.make_weights(synth.DEFAULT_ARCH))
    geo = {}
    t7.load_checkpoint(p, geo)
    assert geo["norm"] == "instance"


def _bn_modules(model):
    from fav_b200 import t7

    out = []

    def walk(m):
        if isinstance(m, t7.T7Object):
            if m.torch_type.endswith("SpatialBatchNormalization"):
                out.append(m)
            for v in m.get("modules", {}).values():
                walk(v)
    walk(model)
    return out


@pytest.mark.parametrize("defect,module", [("mixed", "l3.n1"), ("no_running_var", "l1.n"), ("size", "l2.n")])
def test_bn_checkpoint_geometry_errors_name_the_module(tmp_path, defect, module):
    from fav_b200 import t7

    arch = synth.DEFAULT_ARCH
    p = str(tmp_path / "bn.t7")
    t7.write_checkpoint(p, arch, _bn_weights(arch), reflect_pad=40, norm="batch")
    model = t7.load(p)["model"]
    bns = _bn_modules(model)  # execution order: l0.n, l1.n, l2.n, l3.n1, l3.n2, ...
    if defect == "mixed":
        m = bns[3]
        m.torch_type = "nn.InstanceNormalization"
        m["nOutput"] = 128
    elif defect == "no_running_var":
        del bns[1]["running_var"]
    else:
        bns[2]["running_mean"] = bns[2]["running_mean"][:64]
        bns[2]["running_var"] = bns[2]["running_var"][:64]
    with pytest.raises(t7.GeometryError, match=module.replace(".", r"\.")):
        t7.model_to_state(model)


def test_build_model_honours_use_instance_norm():
    from fav_b200 import models_video

    net = models_video.build_model({"use_instance_norm": 0})
    shapes = net.param_shapes()
    assert net.norm == "batch"
    assert shapes["l0.n.running_mean"] == (32,) and shapes["l0.n.running_var"] == (32,) and shapes["l0.n.eps"] == (1,)
    assert "l0.n.running_mean" not in models_video.build_model({}).param_shapes()


@pytest.mark.parametrize("arch,ptype", ARCHS)
def test_bn_param_table_matches_synth(arch, ptype):
    from fav_b200 import models_video

    net = models_video.StyleNet(arch, padding_type=ptype, norm="batch")
    w = synth.make_weights(arch, "candy", norm="batch")
    shapes = net.param_shapes()
    assert sorted(shapes) == sorted(w)
    for k, shp in shapes.items():
        assert int(np.prod(shp)) == w[k].size, k


def test_unknown_norm_is_refused():
    from fav_b200 import _lib, models_video

    with pytest.raises(_lib.FavError, match="norm must be"):
        models_video.StyleNet(norm="group")


@pytest.mark.parametrize("field,value", [("running_var", -2e-5), ("running_var", np.nan), ("weight", np.inf), ("running_mean", np.nan)])
def test_invalid_bn_statistics_are_refused_at_finalize(field, value):
    """Refused by the host-side folding in fav_net_finalize (FAV_ERR_INVALID, naming the norm), before any device work."""
    from fav_b200 import _lib, models_video

    w = synth.make_weights(synth.DEFAULT_ARCH, "candy", norm="batch")
    w[f"l3.n2.{field}"] = w[f"l3.n2.{field}"].copy()
    w[f"l3.n2.{field}"][5] = value
    net = models_video.StyleNet(norm="batch")
    with pytest.raises(_lib.FavError) as e:
        net.load_state(w)
    assert e.value.status == _lib.FAV_ERR_INVALID and "l3.n2" in str(e.value), str(e.value)


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(EMU, "libfav_emu_opnd_epi.so")
    srcs = [os.path.join(EMU, f) for f in ("opnd_epi_emu.cu", "conv_emu.cu")]
    csrc = os.path.join(ROOT, "fast-artistic-videos_b200", "csrc")
    hdrs = [os.path.join(csrc, h) for h in ("conv_plan.hpp", "conv.cuh", "net_layout.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + hdrs):
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                               "-Wno-deprecated-gpu-targets", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emu_last_error.restype = C.c_char_p
    return lib


def plan_rows(arch, ptype, in_dim=7):
    """The net's layers in execution order as emu_opnd_epi_check reads them (see opnd_epi_emu.cu)."""
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


@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
@pytest.mark.parametrize("arch,ptype", ARCHS)
def test_operand_epilogue_writes_every_interior_element_once(emu, arch, ptype, shape):
    H, W = shape
    rows = plan_rows(arch, ptype)
    R = synth.reflect_start_pad(synth.parse_arch(arch), ptype)
    flat = (C.c_int * (8 * len(rows)))(*[v for r in rows for v in r])
    info = (C.c_int * 4)()
    rc = emu.emu_opnd_epi_check(len(rows), flat, H + 2 * R, W + 2 * R, info)
    assert rc == 0, emu.emu_last_error().decode()
    jobs, parity, phases, nblocks = list(info)
    assert jobs > 0 and parity > 0  # the convs feeding 'd' layers write parity-split operands
    assert phases > 0 or "u" not in arch  # 'u' convs run as 4 sub-pixel phases
    if arch == WIDE:
        assert nblocks > 0  # d256, C256 and f3s1-192 run as two N blocks
