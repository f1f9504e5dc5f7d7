"""-scale_factor on the GPU (fast_artistic_video_core.lua:121-158): the bicubic resampler fav_image_scale_bicubic against the fp64
reading of tests/scale_oracle.py (and bit for bit against its fp32 two-pass form), fav_run_image_scaled against the oracle
composition scale down -> image net -> deprocess -> scale up, its refusals, and `video.main -scale_factor` on a PPM clip."""
import ctypes as C

import numpy as np
import pytest
import torch

import scale_oracle as so
from fav_b200 import _lib, models_video, synth

pytestmark = pytest.mark.gpu

TOL = 1e-3  # the deprocessed-output bar of test_gpu_net.py


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def img_net():
    assert torch.cuda.is_available()
    return models_video.synthetic_model("mosaic", synth.DEFAULT_ARCH, 3)


@pytest.fixture(scope="module")
def img_oracle():
    return so.NetOracle(style="mosaic", dtype=torch.float64, in_dim=3)


def gpu_scale(src, Hout, Wout):
    Cn, Hin, Win = src.shape
    x = T(src.astype(np.float32))
    out = torch.empty((Cn, Hout, Wout), device="cuda")
    _lib.check(_lib.lib.fav_image_scale_bicubic(_lib.dptr(x), _lib.dptr(out), Cn, Hin, Win, Hout, Wout, _lib.stream_ptr()))
    return out.cpu().numpy()


@pytest.mark.parametrize("Cn", [1, 3])
@pytest.mark.parametrize("sizes", [(720, 1280, 360, 640), (97, 75, 48, 37), (64, 96, 96, 144), (37, 53, 37, 106)])
def test_resampler_matches_the_fp64_reading(Cn, sizes):
    Hin, Win, Hout, Wout = sizes
    src = np.random.default_rng(Cn * 1000 + Hin).uniform(-0.2, 1.2, (Cn, Hin, Win)).astype(np.float32)
    got = gpu_scale(src, Hout, Wout)
    ref = so.image_scale_bicubic(src, Hout, Wout)
    err = np.abs(got - ref) / np.maximum(1.0, np.abs(ref))
    assert err.max() <= 2e-6, err.max()
    # the fused kernel is the two-pass form evaluated in fp32, bit for bit
    assert np.array_equal(got, so.image_scale_bicubic_fp32(src, Hout, Wout))
    assert np.array_equal(got[..., -1, -1], src[..., -1, -1])


@pytest.mark.parametrize("H,W,sf", [(128, 192, 0.5), (64, 96, 1.5), (64, 96, 2.0), (720, 1280, 0.5)])
def test_run_image_scaled_vs_oracle_composition(img_net, img_oracle, H, W, sf):
    f = synth.make_frame(H, W, 1)
    out = img_net.run_image(T(f), scale_factor=sf).cpu().numpy()
    ref = img_oracle.run_image(f, scale_factor=sf)
    assert out.shape == (3, H, W)
    assert np.abs(out - ref).max() < TOL / 10
    if H == 64:  # a different stylization from the unscaled one
        assert np.abs(out - img_oracle.run_image(f)).max() > 1e-2


def test_scale_factor_one_is_run_image(img_net):
    H, W = 64, 96
    x = T(synth.make_frame(H, W, 3))
    a, b = torch.empty_like(x), torch.empty_like(x)
    _lib.check(_lib.lib.fav_run_image(img_net._h, _lib.dptr(x), None, H, W, _lib.dptr(a), _lib.stream_ptr()))
    _lib.check(_lib.lib.fav_run_image_scaled(img_net._h, _lib.dptr(x), H, W, C.c_double(1.0), _lib.dptr(b), _lib.stream_ptr()))
    assert torch.equal(a, b)
    assert torch.equal(img_net.run_image(x, scale_factor=1.0), a)


def test_successive_calls_are_bit_identical(img_net):
    """first call eager, second captures the plan's graph, third replays it"""
    H, W = 96, 128
    x = T(synth.make_frame(H, W, 4))
    outs = [img_net.run_image(x, scale_factor=0.5) for _ in range(3)]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])


def test_refusals_before_any_device_work(img_net):
    vid_net = models_video.synthetic_model("candy")
    cases = [(vid_net, 64, 96, 0.5, "separate image model"),  # 7 input channels: core.lua:133-138
             (img_net, 64, 96, 0.3, "integer sides"),  # 19.2 x 28.8
             (img_net, 64, 98, 0.25, "integer sides"),  # w = 24.5
             (img_net, 68, 96, 0.5, "multiples of 4"),  # 34 x 48
             (img_net, 64, 90, 0.5, "multiples of 4")]  # 32 x 45
    for net, H, W, sf, msg in cases:
        x = torch.zeros((3, H, W), device="cuda")
        torch.cuda.synchronize()
        n0 = _lib.lib.fav_launch_count()
        with pytest.raises(_lib.FavError) as e:
            net.run_image(x, scale_factor=sf)
        assert e.value.status == _lib.FAV_ERR_INVALID and msg in e.value.message, (H, W, sf, e.value.message)
        assert _lib.lib.fav_launch_count() == n0
    with pytest.raises(_lib.FavError) as e:  # one image per call
        img_net.run_image(torch.zeros((2, 3, 64, 96), device="cuda"), scale_factor=0.5)
    assert e.value.status == _lib.FAV_ERR_INVALID


def write_clip(d, H, W, n):
    from fav_b200 import consistencyChecker

    for i in range(1, n + 1):
        synth.write_ppm(f"{d}/frame_{i:04d}.ppm", synth.make_frame(H, W, i))
    for i in range(2, n + 1):
        synth.write_flo(f"{d}/backward_{i}_{i - 1}.flo", synth.make_backward_flow(H, W, i))
        synth.write_flo(f"{d}/forward_{i - 1}_{i}.flo", synth.make_forward_flow(H, W, i))
        consistencyChecker.main(["consistencyChecker", f"{d}/backward_{i}_{i - 1}.flo", f"{d}/forward_{i - 1}_{i}.flo",
                                 f"{d}/reliable_{i}_{i - 1}.pgm"])
    return ["-input_pattern", f"{d}/frame_%04d.ppm", "-num_frames", str(n), "-model_vid", "synthetic:candy"]


def read_frame(path):
    from PIL import Image

    return np.asarray(Image.open(path), np.float32).transpose(2, 0, 1) / 255.0


def check_png(path, ref):
    png = read_frame(path)
    assert np.abs(png - np.clip(ref, 0, 1)).max() <= 0.5 / 255 + TOL, path


def test_video_driver_scale_factor(tmp_path, img_oracle):
    """frame 1 from the scaled composition; frames 2-3 from the video model with the upscaled, unclamped frame 1 as the prior
    (fast_artistic_video.lua:169); the recurrence against the oracle's"""
    from fav_b200 import video
    from oracle import net_oracle, pyoracle

    H, W, n = 128, 192, 3
    d = str(tmp_path)
    common = write_clip(d, H, W, n) + ["-model_img", "synthetic:mosaic", "-scale_factor", "0.5"]
    video.main(common + ["-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo", "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm",
                         "-output_prefix", f"{d}/out"])
    vid = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    prev = None
    for i in range(1, n + 1):
        frame = read_frame(f"{d}/frame_{i:04d}.ppm")
        if i == 1:
            ref = img_oracle.run_image(frame, scale_factor=0.5)
        else:
            bw = pyoracle.flo_read(f"{d}/backward_{i}_{i - 1}.flo", 1)
            fw = pyoracle.flo_read(f"{d}/forward_{i - 1}_{i}.flo", 1)
            cert = pyoracle.min_filter(pyoracle.consistency(bw, fw).astype(np.float32) / 255.0, 7)
            ref = vid.run_next_image(frame, prev, synth.checker_to_lua(bw), cert)
        prev = ref.astype(np.float32)
        check_png(f"{d}/out-{i:05d}.png", ref)
    # -create_inconsistent: every frame is a single image through the scaled composition
    video.main(common + ["-create_inconsistent", "-output_prefix", f"{d}/inc"])
    for i in range(1, n + 1):
        check_png(f"{d}/inc-{i:05d}.png", img_oracle.run_image(read_frame(f"{d}/frame_{i:04d}.ppm"), scale_factor=0.5))
    # model_img == nil: the reference's torch.cat of the scaled frame and the unscaled fill fails (core.lua:133-138)
    with pytest.raises(_lib.FavError) as e:
        video.main(write_clip(d, H, W, 1) + ["-model_img", "self", "-scale_factor", "0.5", "-create_inconsistent",
                                            "-output_prefix", f"{d}/self"])
    assert e.value.status == _lib.FAV_ERR_INVALID
