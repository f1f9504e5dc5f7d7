"""Stylization nets with layers wider than 128 channels (N-blocked conv_tc_kernel jobs, fused InstanceNorm statistics per block,
norm-on-load per block) vs the fp64 PyTorch oracle, through the C ABI, the frame loop, the host-buffer session and a .t7
checkpoint.  Bars as in test_gpu_net.py: 2e-4 * max|ref| per layer, TOL / 10 on the deprocessed frame."""
import numpy as np
import pytest
import torch

from fav_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3
DOUBLED = "c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3"               # the default arch at twice the width, two residual blocks
DOUBLED_PAPER = "c9s1-64,d128,d256,R256,R256,U2,c3s1-128,U2,c9s1-3"   # the paper arch at twice the width


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rand_input(H, W, seed=0, in_dim=7):
    from oracle import pyoracle

    rng = np.random.default_rng(seed)
    x7 = pyoracle.first_frame_input(synth.make_frame(H, W, 1))
    x7[3:6] = rng.normal(0, 50, (3, H, W))
    x7[6] = rng.uniform(0, 1, (H, W))
    return x7[:in_dim].astype(np.float32)


@pytest.fixture(scope="module")
def doubled():
    from fav_b200 import models_video

    return models_video.synthetic_model("candy", DOUBLED)


# 48x508: output widths of the residual convs cross 128-pixel tile edges
@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
@pytest.mark.parametrize("arch,ptype,in_dim", [
    (DOUBLED, "reflect-start", 7),
    (DOUBLED_PAPER, "reflect-start", 7),                                # U2 on 256 channels; final x-fold conv from 128
    ("c9s1-144,d208,d384,R384,u208,u128,c9s1-3", "reflect-start", 7),  # partial last blocks, 3 blocks, R384 via in_apply
    ("c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3", "reflect-start", 7),  # wide CX block, wide stride-1 full conv
    (DOUBLED, "zero", 7),                                               # padded residual convs, Identity skip
    (DOUBLED, "reflect-start", 3),                                      # 3-channel image model
])
def test_wide_arch_every_layer_vs_fp64_oracle(arch, ptype, in_dim, shape):
    from fav_b200 import models_video
    from oracle import net_oracle

    H, W = shape
    w = synth.make_weights(arch, "scream", in_dim)
    net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim).load_state(w)
    ora = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=in_dim)
    x = rand_input(H, W, 9, in_dim)
    taps = {}
    ref = ora.forward(torch.from_numpy(x)[None], taps)[0].numpy()
    out = net.forward(T(x)[None]).cpu().numpy()[0]
    assert out.shape == ref.shape == (3, H, W)
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = net.layer_output(i).cpu().numpy()
        assert g.shape == r.shape and np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"layer {i}"
    assert np.abs(out - ref).max() / 255.0 < TOL / 10
    f1 = synth.make_frame(H, W, 1)
    assert np.abs(net.run_image(T(f1)).cpu().numpy() - ora.run_image(f1)).max() < TOL / 10


def test_wide_recurrence_vs_oracle_clip(doubled):
    """3 frames of run_image / run_next_image at 128x200 (the GPU's own trajectory) vs net_oracle.run_clip."""
    from oracle import net_oracle

    H, W = 128, 200
    ora = net_oracle.NetOracle(arch=DOUBLED, style="candy", dtype=torch.float64)
    ref = net_oracle.run_clip(ora, H, W, 3)
    prev = None
    for i in range(1, 4):
        frame = T(synth.make_frame(H, W, i))
        if i == 1:
            out = doubled.run_image(frame)
        else:
            flow = T(synth.checker_to_lua(synth.make_backward_flow(H, W, i)))
            out = doubled.run_next_image(frame, prev, flow, T(net_oracle.make_cert(H, W, i)))
        err = float(np.abs(out.cpu().numpy() - ref[i - 1]).max())
        assert err < TOL / 10, (i, err)
        prev = out


def test_wide_tcgen05_agrees_with_cuda_core_comparator(doubled):
    x = T(rand_input(96, 160, 3))[None]
    a = doubled.forward(x)
    doubled.set_conv_impl("simt")
    try:
        b = doubled.forward(x)
    finally:
        doubled.set_conv_impl("tcgen05")
    assert float((a - b).abs().max()) / 255.0 < 5e-5


def test_wide_session_host_buffers_match_device_api(doubled):
    from fav_b200 import consistencyChecker, session, utils

    H, W = 96, 128
    s = session.Session(doubled, H, W)
    frames = [torch.from_numpy(synth.make_frame(H, W, i)).pin_memory() for i in range(1, 4)]
    outs = [torch.empty((3, H, W)).pin_memory() for _ in range(3)]
    s.run_image(frames[0], outs[0])
    for i in range(2, 4):
        bw = torch.from_numpy(synth.make_backward_flow(H, W, i)).pin_memory()
        fw = torch.from_numpy(synth.make_forward_flow(H, W, i)).pin_memory()
        s.run_next_image_flows(frames[i - 1], bw, fw, outs[i - 1], 7)
    s.sync()
    prev = doubled.run_image(frames[0].cuda())
    assert torch.equal(prev.cpu(), outs[0])
    for i in range(2, 4):
        bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
        _, cert = consistencyChecker.check(T(bw), T(fw), want_cert=True)
        prev = doubled.run_next_image(frames[i - 1].cuda(), prev, T(synth.checker_to_lua(bw)), utils.min_filter(cert, 7))
        assert torch.equal(prev.cpu(), outs[i - 1]), i


def test_wide_t7_checkpoint_loads_and_runs(tmp_path):
    from fav_b200 import core, t7
    from oracle import net_oracle

    H, W = 64, 96
    w = synth.make_weights(DOUBLED, "mosaic")
    p = str(tmp_path / "wide.t7")
    t7.write_checkpoint(p, DOUBLED, w, reflect_pad=synth.reflect_start_pad(synth.parse_arch(DOUBLED, 7)))
    net = core.load_model(p)
    assert net.arch == DOUBLED
    f1 = synth.make_frame(H, W, 1)
    ref = net_oracle.NetOracle(arch=DOUBLED, style="mosaic", dtype=torch.float64).run_image(f1)
    assert np.abs(net.run_image(T(f1)).cpu().numpy() - ref).max() < TOL / 10


def test_wide_720p_forward_vs_fp64_oracle(doubled):
    """One 1280x720 frame of the doubled default arch; the fp64 oracle needs tens of seconds on the CPU."""
    from oracle import net_oracle

    H, W = 720, 1280
    f1 = synth.make_frame(H, W, 1)
    out = doubled.run_image(T(f1)).cpu().numpy()
    ref = net_oracle.NetOracle(arch=DOUBLED, style="candy", dtype=torch.float64).run_image(f1)
    assert np.abs(out - ref).max() < TOL / 10
