"""Batch-normalized stylization nets (-use_instance_norm 0) on the GPU: BatchNorm folded into the convolutions, each non-final
conv_tc_kernel job writing the next operand from its accumulators (operand epilogue).  Compared with the fp64 oracle
(tests/bn_oracle.py) on running statistics calibrated to the net's own activations.  Bars as in test_gpu_net.py /
test_gpu_wide_net.py: 2e-4 * max|ref| per layer, TOL / 10 on the deprocessed frame."""
import functools

import numpy as np
import pytest
import torch

import bn_oracle
from fav_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3
WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"  # N blocks, a CX block, an f token, a parity-split consumer


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def weights(arch, ptype="reflect-start", in_dim=7, style="candy"):
    return bn_oracle.calibrate_bn_weights(arch, style, in_dim, 64, 96, padding_type=ptype)


def make_net(arch, ptype="reflect-start", in_dim=7):
    from fav_b200 import models_video

    return models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim, norm="batch").load_state(weights(arch, ptype, in_dim))


def make_oracle(arch, ptype="reflect-start", in_dim=7):
    return bn_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=weights(arch, ptype, in_dim), padding_type=ptype, in_dim=in_dim)


@pytest.fixture(scope="module")
def default_net():
    return make_net(synth.DEFAULT_ARCH)


# 48x508: output widths of the residual convs cross 128-pixel tile edges
@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
@pytest.mark.parametrize("arch,ptype", [
    (synth.DEFAULT_ARCH, "reflect-start"),
    (synth.DEFAULT_ARCH, "zero"),      # padded residual convs, Identity skip
    (synth.PAPER_ARCH, "reflect-start"),  # U2: the BN after the upsampling is not folded
    (WIDE, "reflect-start"),
])
def test_bn_arch_every_layer_vs_fp64_oracle(arch, ptype, shape):
    H, W = shape
    net, ora = make_net(arch, ptype), make_oracle(arch, ptype)
    x = bn_oracle.calibration_input(H, W, seed=9)
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


def test_bn_image_model_run_image():
    """A separate 3-channel image model (-model_img)."""
    H, W = 64, 96
    net, ora = make_net(synth.DEFAULT_ARCH, in_dim=3), make_oracle(synth.DEFAULT_ARCH, in_dim=3)
    f1 = synth.make_frame(H, W, 1)
    assert np.abs(net.run_image(T(f1)).cpu().numpy() - ora.run_image(f1)).max() < TOL / 10


def test_bn_recurrence_vs_oracle_clip(default_net):
    """3 frames of run_image / run_next_image (the GPU's own trajectory) vs net_oracle.run_clip."""
    from oracle import net_oracle

    H, W = 128, 200
    ref = net_oracle.run_clip(make_oracle(synth.DEFAULT_ARCH), H, W, 3)
    prev = None
    for i in range(1, 4):
        frame = T(synth.make_frame(H, W, i))
        if i == 1:
            out = default_net.run_image(frame)
        else:
            flow = T(synth.checker_to_lua(synth.make_backward_flow(H, W, i)))
            out = default_net.run_next_image(frame, prev, flow, T(net_oracle.make_cert(H, W, i)))
        err = float(np.abs(out.cpu().numpy() - ref[i - 1]).max())
        assert err < TOL / 10, (i, err)
        prev = out


@pytest.mark.parametrize("arch", [synth.DEFAULT_ARCH, synth.PAPER_ARCH, WIDE])
def test_bn_tensor_core_agrees_with_cuda_core_comparator(arch):
    """The comparator writes raw fp32 and packs through in_apply without normalisation; the tensor-core path packs in the
    conv epilogue."""
    net = make_net(arch)
    x = T(bn_oracle.calibration_input(96, 160, seed=3))[None]
    a = net.forward(x)
    net.set_conv_impl("simt")
    try:
        b = net.forward(x)
    finally:
        net.set_conv_impl("tcgen05")
    assert float((a - b).abs().max()) / 255.0 < 5e-5
    assert torch.equal(net.forward(x), a)  # the tensor-core path after a comparator run (lazily allocated raw tensors)


def test_bn_repeats_are_bit_identical(default_net):
    """No atomics on the BN path: the same frame gives the same bits, eagerly and through the captured graph."""
    H, W = 136, 240
    x = T(bn_oracle.calibration_input(H, W, seed=5))[None]
    outs = [default_net.forward(x) for _ in range(3)]
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    f = T(synth.make_frame(H, W, 1))
    imgs = [default_net.run_image(f) for _ in range(4)]  # eager, capture, graph launches
    assert all(torch.equal(o, imgs[0]) for o in imgs[1:])


def test_bn_t7_checkpoint_through_video_main(tmp_path):
    """A BN checkpoint written by write_checkpoint(norm='batch') through `video.main -model_vid x.t7`."""
    from PIL import Image

    from fav_b200 import consistencyChecker, t7, video
    from oracle import pyoracle

    H, W, n = 64, 96, 3
    d = str(tmp_path)
    for i in range(1, n + 1):
        synth.write_ppm(f"{d}/frame_{i:04d}.ppm", synth.make_frame(H, W, i))
    for i in range(2, n + 1):
        synth.write_flo(f"{d}/backward_{i}_{i - 1}.flo", synth.make_backward_flow(H, W, i))
        synth.write_flo(f"{d}/forward_{i - 1}_{i}.flo", synth.make_forward_flow(H, W, i))
        consistencyChecker.main(["consistencyChecker", f"{d}/backward_{i}_{i - 1}.flo", f"{d}/forward_{i - 1}_{i}.flo",
                                 f"{d}/reliable_{i}_{i - 1}.pgm"])
    t7.write_checkpoint(f"{d}/bn.t7", synth.DEFAULT_ARCH, weights(synth.DEFAULT_ARCH), norm="batch")
    video.main(["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo",
                "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-model_vid", f"{d}/bn.t7",
                "-output_prefix", f"{d}/out", "-num_frames", str(n)])
    ora = make_oracle(synth.DEFAULT_ARCH)
    prev = None
    for i in range(1, n + 1):
        frame = np.asarray(Image.open(f"{d}/frame_{i:04d}.ppm"), np.float32).transpose(2, 0, 1) / 255.0
        if i == 1:
            ref = ora.run_image(frame)
        else:
            bw = pyoracle.flo_read(f"{d}/backward_{i}_{i - 1}.flo", 1)
            fw = pyoracle.flo_read(f"{d}/forward_{i - 1}_{i}.flo", 1)
            cert = pyoracle.min_filter(pyoracle.consistency(bw, fw).astype(np.float32) / 255.0, 7)
            ref = ora.run_next_image(frame, prev, synth.checker_to_lua(bw), cert)
        prev = ref.astype(np.float32)
        png = np.asarray(Image.open(f"{d}/out-{i:05d}.png"), np.float32).transpose(2, 0, 1) / 255.0
        assert np.abs(png - np.clip(ref, 0, 1)).max() <= 0.5 / 255 + TOL, i


def test_bn_720p_frame_vs_fp64_oracle(default_net):
    """One 1280x720 frame of the default arch; the fp64 oracle needs tens of seconds on the CPU."""
    H, W = 720, 1280
    f1 = synth.make_frame(H, W, 1)
    out = default_net.run_image(T(f1)).cpu().numpy()
    assert np.abs(out - make_oracle(synth.DEFAULT_ARCH).run_image(f1)).max() < TOL / 10
