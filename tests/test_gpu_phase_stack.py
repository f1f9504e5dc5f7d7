"""Stacked sub-pixel phases on the GPU: the default arch's two stride-2 transposed convs run with their phases stacked along
the MMA's N (u64: two jobs of N = 128, u32: one job of N = 128 that normalises u64's output on load) instead of one job per
phase (FAV_NO_STACK=1).  Every layer is bit-identical to the per-phase plan's, also over recurrent frames, and within the
fp64-oracle bars of test_gpu_nl_fusion.py; a batch is bit-identical to its images run alone, and the norm-on-load plan to
the plan with every pass run (FAV_NO_NL=1), with the phases stacked."""
import os

import pytest
import torch

from fav_b200 import synth
from test_gpu_net import TOL, T, rand_input

pytestmark = pytest.mark.gpu

ARCH = synth.DEFAULT_ARCH
NTOK = len(synth.parse_arch(ARCH))


def make_net(ptype):
    from fav_b200 import models_video

    return models_video.StyleNet(ARCH, padding_type=ptype).load_state(synth.make_weights(ARCH, "scream", 7))


def planned_with(env, ptype, fn):
    """fn(net) on a fresh net whose plans are built with the variables `env` set (they are read when a plan is built, at a
    net's first call at each size)."""
    keys = ("FAV_NO_STACK", "FAV_NO_NL")
    old = {k: os.environ.pop(k, None) for k in keys}
    os.environ.update(env)
    try:
        return fn(make_net(ptype))
    finally:
        for k in keys:
            os.environ.pop(k, None)
            if old[k] is not None:
                os.environ[k] = old[k]


def forward_layers(x):
    def fn(net):
        from fav_b200 import _lib

        net.forward(x)  # builds the plan
        n0 = _lib.lib.fav_launch_count()
        y = net.forward(x)
        torch.cuda.synchronize()
        launches = _lib.lib.fav_launch_count() - n0
        layers = [[net.layer_output(i, b) for i in range(NTOK - 1)] for b in range(x.size(0))]
        torch.cuda.synchronize()
        return y, layers, launches
    return fn


@pytest.mark.parametrize("shape", [(64, 96), (48, 508), (720, 1280)])
@pytest.mark.parametrize("ptype", ["reflect-start", "zero"])
def test_default_arch_stacked_vs_per_phase_and_fp64(ptype, shape):
    from oracle import net_oracle

    H, W = shape
    x7 = rand_input(H, W, 3)
    x = T(x7)[None]
    yp, lp, np_launch = planned_with({"FAV_NO_STACK": "1"}, ptype, forward_layers(x))
    ys, ls, ns_launch = planned_with({}, ptype, forward_layers(x))
    assert np_launch - ns_launch == 5  # u64: 4 phase jobs -> 2, u32: 4 -> 1
    for i, (p, s) in enumerate(zip(lp[0], ls[0])):  # zero weights add exact zeros, each phase's statistics flush separately
        assert torch.equal(p, s), f"layer {i}: {(s - p).abs().max().item()}"
    assert torch.equal(ys, yp)
    ora = net_oracle.NetOracle(arch=ARCH, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=7)
    ora.w = {k: v.cuda() for k, v in ora.w.items()}
    taps = {}
    ref = ora.forward(torch.from_numpy(x7)[None].cuda(), taps)[0]
    for i in range(NTOK - 1):
        r = taps[f"l{i}"][0]
        assert (ls[0][i].double() - r).abs().max().item() < 2e-4 * max(1.0, r.abs().max().item()), f"layer {i}"
    assert (ys[0].double() - ref).abs().max().item() / 255.0 < TOL / 10


def test_batch_of_three_bit_identical_to_each_image():
    xs = [T(rand_input(64, 96, s))[None] for s in (6, 7, 8)]
    yb, lb, _ = planned_with({}, "reflect-start", forward_layers(torch.cat(xs)))
    for b, x in enumerate(xs):
        y1, l1, _ = planned_with({}, "reflect-start", forward_layers(x))
        assert torch.equal(yb[b], y1[0]), f"image {b}"
        for i, (p, q) in enumerate(zip(lb[b], l1[0])):
            assert torch.equal(p, q), f"image {b} layer {i}"


def test_norm_on_load_bit_identical_with_stacking():
    x = T(rand_input(64, 96, 5))[None]
    ya, la, na = planned_with({"FAV_NO_NL": "1"}, "reflect-start", forward_layers(x))
    yb, lb, nb = planned_with({}, "reflect-start", forward_layers(x))
    assert na > nb  # the folded passes do not run
    assert torch.equal(ya, yb)
    for i, (p, q) in enumerate(zip(la[0], lb[0])):
        assert torch.equal(p, q), f"layer {i}"


def test_recurrent_720p_frames_bit_identical_to_per_phase():
    """run_image, then run_next_image frames fed back through the cached graph: errors would compound from frame to frame."""
    from oracle import net_oracle

    H, W = 720, 1280
    f1, f2 = T(synth.make_frame(H, W, 1)), T(synth.make_frame(H, W, 2))
    flow = T(synth.checker_to_lua(synth.make_backward_flow(H, W, 2)))
    cert = T(net_oracle.make_cert(H, W, 2))

    def fn(net):
        prev = net.run_image(f1)
        frames = [prev]
        for _ in range(6):  # eager, capture, graph replays
            prev = net.run_next_image(f2, prev, flow, cert)
            frames.append(prev)
        torch.cuda.synchronize()
        return frames

    fp = planned_with({"FAV_NO_STACK": "1"}, "reflect-start", fn)
    fs = planned_with({}, "reflect-start", fn)
    for i, (p, s) in enumerate(zip(fp, fs)):
        assert torch.equal(p, s), f"frame {i}: {(s - p).abs().max().item()}"
