"""Norm-on-load on the GPU: a net whose InstanceNorm passes are folded into the convolutions that read them (the stride-2
convs, the sub-pixel phase jobs of transposed convs, the second conv of every block, plain convs) computes
exactly what the same net computes with every pass run on its own (FAV_NO_NL=1): the final frame and every arch token's
activation (fav_net_layer_output, which replays the forward with a folded pass run) are bit-identical, single image, batched
and on the recurrent frame path at 720p.  The fp64 oracle bars of test_gpu_net.py hold for the fused net."""
import os

import numpy as np
import pytest
import torch

from fav_b200 import synth
from test_gpu_net import TOL, T, rand_input

pytestmark = pytest.mark.gpu


def make_net(arch, ptype, style="scream"):
    from fav_b200 import models_video

    return models_video.StyleNet(arch, padding_type=ptype).load_state(synth.make_weights(arch, style, 7))


def run_pair(arch, ptype, fn):
    """fn(net) on a net planned with every pass separate (FAV_NO_NL=1) and on the same net planned with norm-on-load.  Plans
    are built (and FAV_NO_NL read) at a net's first call at each size, so the environment only has to hold during fn."""
    out = []
    for no_nl in (True, False):
        net = make_net(arch, ptype)
        old = os.environ.pop("FAV_NO_NL", None)
        if no_nl:
            os.environ["FAV_NO_NL"] = "1"
        try:
            out.append(fn(net))
        finally:
            os.environ.pop("FAV_NO_NL", None)
            if old is not None:
                os.environ["FAV_NO_NL"] = old
    return out


def forward_and_layers(x, ntok):
    def fn(net):
        y = net.forward(x)
        layers = [[net.layer_output(i, b) for i in range(ntok - 1)] for b in range(x.size(0))]
        # a second read of each layer after the replays: still today's bits, and the frame a forward computes is unchanged
        again = net.layer_output(0, 0)
        y2 = net.forward(x)
        torch.cuda.synchronize()
        return y, layers, again, y2, net.profile(x[:1]) if x.size(0) == 1 else None
    return fn


def assert_same(a, b):
    ya, la, ga, y2a, pa = a
    yb, lb, gb, y2b, pb = b
    assert torch.equal(ya, yb)
    assert torch.equal(y2a, yb) and torch.equal(y2b, yb)
    for ib, (ia_l, ib_l) in enumerate(zip(la, lb)):
        for i, (p, q) in enumerate(zip(ia_l, ib_l)):
            assert torch.equal(p, q), f"image {ib} layer {i}"
    assert torch.equal(ga, la[0][0]) and torch.equal(gb, lb[0][0])
    if pa is not None:  # the fused plan drops in_apply passes and nothing else
        na = sum(r["kind"] == "in_apply" for r in pa)
        nb = sum(r["kind"] == "in_apply" for r in pb)
        assert nb < na
        assert [r["name"] for r in pa if r["kind"] == "conv"] == [r["name"] for r in pb if r["kind"] == "conv"]


@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
@pytest.mark.parametrize("ptype", ["reflect-start", "zero"])
def test_default_arch_bit_identical_and_vs_fp64(ptype, shape):
    from oracle import net_oracle

    H, W = shape
    arch = synth.DEFAULT_ARCH
    x7 = rand_input(H, W, 3)
    a, b = run_pair(arch, ptype, forward_and_layers(T(x7)[None], len(synth.parse_arch(arch))))
    assert_same(a, b)
    ora = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=7)
    taps = {}
    ref = ora.forward(torch.from_numpy(x7)[None], taps)[0].numpy()
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = b[1][0][i].cpu().numpy()
        assert np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"layer {i}"
    assert np.abs(b[0].cpu().numpy()[0] - ref).max() / 255.0 < TOL / 10


def test_default_arch_folds_eight_passes():
    """The passes after l0 and d64 (read by the stride-2 convs), after u64 (read by u32's four sub-pixel phase jobs) and the
    inner pass of each residual block.  The block outputs (skip adds), the pass after d128 (the first block's skip) and the
    pass after u32 (read by the x-fold final conv, which runs slower fused) stay."""
    arch = synth.DEFAULT_ARCH
    x = T(rand_input(64, 96, 5))[None]
    a, b = run_pair(arch, "reflect-start", lambda net: net.profile(x))
    names = lambda p: [r["name"] for r in p if r["kind"] == "in_apply"]
    assert set(names(a)) - set(names(b)) == {"l0.n.apply", "l1.n.apply", "l8.n.apply"} | {f"l{i}.n1.apply" for i in range(3, 8)}
    assert names(b) == ["l2.n.apply"] + [f"l{i}.n2.apply" for i in range(3, 8)] + ["l9.n.apply"]


def test_paper_arch_bit_identical():
    arch = synth.PAPER_ARCH
    x7 = rand_input(64, 96, 4)
    a, b = run_pair(arch, "reflect-start", forward_and_layers(T(x7)[None], len(synth.parse_arch(arch))))
    assert_same(a, b)


def test_batch_of_three_bit_identical():
    arch = synth.DEFAULT_ARCH
    x = T(np.stack([rand_input(64, 96, s) for s in (6, 7, 8)]))
    a, b = run_pair(arch, "reflect-start", forward_and_layers(x, len(synth.parse_arch(arch))))
    assert_same(a, b)


def test_720p_frame_and_recurrent_frames_bit_identical():
    """One 720p forward with every layer, then three recurrent run_next_image frames through the cached graph."""
    from oracle import net_oracle

    arch = synth.DEFAULT_ARCH
    H, W = 720, 1280
    x = T(rand_input(H, W, 9))[None]
    f1, f2 = T(synth.make_frame(H, W, 1)), T(synth.make_frame(H, W, 2))
    flow = T(synth.checker_to_lua(synth.make_backward_flow(H, W, 2)))
    cert = T(net_oracle.make_cert(H, W, 2))

    def fn(net):
        res = forward_and_layers(x, len(synth.parse_arch(arch)))(net)
        prev = net.run_image(f1)
        frames = [prev]
        for _ in range(3):  # eager, capture, graph replay
            prev = net.run_next_image(f2, prev, flow, cert)
            frames.append(prev)
        torch.cuda.synchronize()
        return res, frames

    (ra, fa), (rb, fb) = run_pair(arch, "reflect-start", fn)
    assert_same(ra, rb)
    for i, (p, q) in enumerate(zip(fa, fb)):
        assert torch.equal(p, q), f"frame {i}"
