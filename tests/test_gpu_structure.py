"""The checker's 4-argument mode inside the frame (fav_run_next_image_flows_structure and the session call): the corners of the
frame being stylized, their exact parallel average and the fused temporal stage (MODE 2), bit for bit against the oracle, the
reference binary's masks and the standalone composition fav_compute_corners -> fav_consistency_check -> cert-given run."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from fav_b200 import synth

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden  # noqa: E402
import make_structure_golden  # noqa: E402


@pytest.fixture(scope="module")
def fav():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    import fav_b200
    from fav_b200 import consistencyChecker, models_video, session  # noqa: F401

    return fav_b200


@pytest.fixture(scope="module")
def net(fav):
    return fav.models_video.synthetic_model("candy")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def content_of(img255):
    """image.load's byte/255 of the frame whose 0..255 planes the checker read."""
    return (img255 / np.float32(255.0)).astype(np.float32)


def ref_avg(corners):
    from oracle import pyoracle

    return float(pyoracle.lib().orc_avg(corners.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(corners.size)))


def frame_case(H, W, idx, seed):
    bw, fw, _, img255 = make_golden.consistency_inputs(H, W, idx, 0.5, seed)
    return bw, fw, img255


@pytest.mark.parametrize("shape", [(64, 96), (100, 76), (97, 75), (256, 256), (240, 320), (720, 1280), (1080, 1920),
                                   (2048, 2048), (2160, 3840)])
def test_compute_corners_and_average(fav, shape):
    from oracle import pyoracle

    H, W = shape
    _, _, _, img255 = make_golden.consistency_inputs(H, W, 2, 0.6, 5)
    corners, avg = fav.consistencyChecker.compute_corners(T(img255))
    o = pyoracle.compute_corners(img255)
    assert np.array_equal(corners.cpu().numpy(), o)
    assert np.float32(avg.item()).tobytes() == np.float32(ref_avg(o)).tobytes()


def test_average_of_negative_corners(fav):
    """normalize's `else if` quirk leaves the first corners below the minimum: the exact average handles negative elements."""
    from oracle import pyoracle

    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, size=(3, 200, 300)).astype(np.float32)
    img[:, :20, :20] = 90.0
    o = pyoracle.compute_corners(img)
    assert (o < 0).any()
    corners, avg = fav.consistencyChecker.compute_corners(T(img))
    assert np.array_equal(corners.cpu().numpy(), o)
    assert np.float32(avg.item()).tobytes() == np.float32(ref_avg(o)).tobytes()


def run_structure(net, img255, prev, bw, fw, r, unaligned=False):
    flow = synth.checker_to_lua(bw)
    tflow = T(flow)
    if unaligned:  # a plane one float off 16-byte alignment: the unfused kernels
        buf = torch.empty(flow.size + 1, device="cuda")
        buf[1:] = tflow.reshape(-1)
        tflow = buf[1:].view(flow.shape)
    return net.run_next_image_flows_structure(T(content_of(img255)), T(prev), tflow, T(fw), r)


def run_given(net, img255, prev, bw, cert, r):
    return net.run_next_image_flows(T(content_of(img255)), T(prev), T(synth.checker_to_lua(bw)), None, T(cert), r)


def golden_cases():  # frames the net takes: H, W multiples of 4 and above its reflection padding
    cases = [("consistency", c) for c in make_golden.CONSISTENCY_CASES if c[0] % 4 == 0 and c[1] % 4 == 0]
    return cases + [("structure", "const_64x96")]


@pytest.mark.parametrize("name", list(make_structure_golden.STRUCTURE_CASES))
def test_standalone_check_equals_reference_binary(fav, name):
    """fav_compute_corners (exact average) -> fav_consistency_check on the constant and the 16 x 16 frame."""
    g = np.load(os.path.join(ROOT, "tests", "golden", f"structure_{name}.npz"))
    H, W = (int(v) for v in g["shape"])
    ref4 = np.unpackbits(g["ref4"])[: H * W].reshape(H, W).astype(np.uint8) * 255
    bw, fw, _, img255 = make_structure_golden.structure_inputs(name)
    assert np.array_equal(fav.consistencyChecker.check(T(bw), T(fw), T(img255)).cpu().numpy(), ref4)


@pytest.mark.parametrize("kind,case", golden_cases())
@pytest.mark.parametrize("unaligned", [False, True])
def test_fused_certainty_equals_reference_binary(fav, net, kind, case, unaligned):
    """The 4-argument certainty of the fused stage (and of its unfused fallback) is the reference binary's mask: the frame run
    with it is bit-identical to the frame run with min_filter(ref4 / 255) given."""
    if kind == "consistency":
        H, W, idx, sigma, seed = case
        g = np.load(os.path.join(ROOT, "tests", "golden", f"consistency_{H}x{W}.npz"))
        bw, fw, _, img255 = make_golden.consistency_inputs(H, W, idx, sigma, seed)
    else:
        g = np.load(os.path.join(ROOT, "tests", "golden", f"structure_{case}.npz"))
        H, W = (int(v) for v in g["shape"])
        bw, fw, _, img255 = make_structure_golden.structure_inputs(case)
    ref4 = np.unpackbits(g["ref4"])[: H * W].reshape(H, W).astype(np.float32)
    prev = synth.make_frame(H, W, 1) * 1.2 - 0.1
    for r in (7, 1):
        out = run_structure(net, img255, prev, bw, fw, r, unaligned)
        assert torch.equal(out, run_given(net, img255, prev, bw, ref4, r)), (case, r)


def test_fused_certainty_equals_oracle_720p(fav, net):
    from oracle import pyoracle

    H, W = 720, 1280
    bw, fw, img255 = frame_case(H, W, 3, 8)
    prev = synth.make_frame(H, W, 2)
    cert = pyoracle.consistency(bw, fw, img255).astype(np.float32) / 255.0
    assert (cert != pyoracle.consistency(bw, fw).astype(np.float32) / 255.0).any()  # the structure term matters here
    assert torch.equal(run_structure(net, img255, prev, bw, fw, 7), run_given(net, img255, prev, bw, cert, 7))


def composition(fav, net, img255, prev_t, bw, fw, r):
    """fav_compute_corners -> fav_consistency_check -> fav_run_next_image_flows(cert_raw)."""
    _, cert = fav.consistencyChecker.check(T(bw), T(fw), T(img255), want_cert=True)
    return net.run_next_image_flows(T(content_of(img255)), prev_t, T(synth.checker_to_lua(bw)), None, cert, r)


@pytest.mark.parametrize("shape", [(64, 96), (240, 320), (720, 1280)])
def test_recurrence_equals_composition(fav, net, shape):
    H, W = shape
    frames = 1 if H == 720 else 3
    p_new = p_ref = T(synth.make_frame(H, W, 1))
    for i in range(frames):
        bw, fw, img255 = frame_case(H, W, 2 + i, 20 + i)
        a = net.run_next_image_flows_structure(T(content_of(img255)), p_new, T(synth.checker_to_lua(bw)), T(fw), 7)
        b = composition(fav, net, img255, p_ref, bw, fw, 7)
        assert torch.equal(a, b), (shape, i)
        p_new, p_ref = a, b


def test_three_argument_run_unchanged_after_four_argument_run(fav, net):
    H, W = 64, 96
    bw, fw, img255 = frame_case(H, W, 2, 31)
    x, p, f = T(content_of(img255)), T(synth.make_frame(H, W, 1)), T(synth.checker_to_lua(bw))
    before = net.run_next_image_flows(x, p, f, T(fw), None, 7).clone()
    net.run_next_image_flows_structure(x, p, f, T(fw), 7)
    after = net.run_next_image_flows(x, p, f, T(fw), None, 7)
    assert torch.equal(before, after)


def test_session_equals_composition(fav, net):
    H, W = 64, 96
    s = fav.session.Session(net, H, W)
    first = synth.make_frame(H, W, 1)
    out = np.empty((3, H, W), np.float32)
    s.run_image(first, out)
    s.sync()
    prev_ref = T(out.copy())
    for i in range(3):
        bw, fw, img255 = frame_case(H, W, 2 + i, 40 + i)
        s.run_next_image_flows_structure(content_of(img255), np.ascontiguousarray(bw), np.ascontiguousarray(fw), out)
        s.sync()
        ref = composition(fav, net, img255, prev_ref, bw, fw, 7)
        assert np.array_equal(out, ref.cpu().numpy()), i
        prev_ref = ref


def test_refusals(fav, net):
    from fav_b200 import _lib

    z = torch.zeros((3, 2, 2), device="cuda")
    with pytest.raises(_lib.FavError) as e:
        net.run_next_image_flows_structure(z, z, z[:2], z[:2], 7)
    assert e.value.status == _lib.FAV_ERR_INVALID
    H, W = 64, 96
    x = torch.zeros((3, H, W), device="cuda")
    with pytest.raises(_lib.FavError) as e:
        net.run_next_image_flows_structure(x, x, x[:2], x[:2], 4)
    assert e.value.status == _lib.FAV_ERR_INVALID


def write_clip(d, H, W, n):
    """PPM frames, backward / forward .flo files and the oracle's 4-argument PGMs (frame i as the checker's image)."""
    from fav_b200 import consistencyChecker
    from oracle import pyoracle

    for i in range(1, n + 1):
        fr = synth.make_frame(H, W, i)
        fr[:, :, : W // 2] = 0.5  # a flat half: the structure term matters there
        synth.write_ppm(f"{d}/frame_{i:04d}.ppm", fr)
    for i in range(2, n + 1):
        bw = synth.make_backward_flow(H, W, i)
        fw = (synth.make_forward_flow(H, W, i) + np.random.default_rng(i).normal(0, 0.5, size=(2, H, W))).astype(np.float32)
        synth.write_flo(f"{d}/backward_{i}_{i - 1}.flo", bw)
        synth.write_flo(f"{d}/forward_{i - 1}_{i}.flo", fw)
        img255 = consistencyChecker.read_ppm_planes(f"{d}/frame_{i:04d}.ppm")
        rel = pyoracle.consistency(bw, fw, img255)
        open(f"{d}/reliable_{i}_{i - 1}.pgm", "wb").write(b"P5\n%d %d\n255\n" % (W, H) + rel.tobytes())


def test_bytes_path_equals_composition(fav, net, tmp_path):
    """fav_session_run_frame_bytes_flows (two .flo payloads, no PGM) == fav_session_run_frame_bytes given the 4-argument mask."""
    from fav_b200 import consistencyChecker, flowFileLoader

    H, W, n = 64, 96, 4
    d = str(tmp_path)
    write_clip(d, H, W, n)
    sa, sb = fav.session.Session(net, H, W), fav.session.Session(net, H, W)
    ra, rb = np.empty((H, 1 + 3 * W), np.uint8), np.empty((H, 1 + 3 * W), np.uint8)
    for i in range(1, n + 1):
        rgb = np.ascontiguousarray(np.transpose(consistencyChecker.read_ppm_planes(f"{d}/frame_{i:04d}.ppm"), (1, 2, 0))
                                   .astype(np.uint8))
        if i == 1:
            sa.run_frame_bytes_flows(rgb, None, None, ra)
            sb.run_frame_bytes(rgb, None, None, rb)
        else:
            bw = np.ascontiguousarray(flowFileLoader.load(f"{d}/backward_{i}_{i - 1}.flo", layout=1).transpose(1, 2, 0))
            fw = np.ascontiguousarray(flowFileLoader.load(f"{d}/forward_{i - 1}_{i}.flo", layout=1).transpose(1, 2, 0))
            cert8 = synth.read_pgm(f"{d}/reliable_{i}_{i - 1}.pgm")
            assert (cert8 == 0).any() and (cert8 == 255).any()
            sa.run_frame_bytes_flows(rgb, bw, fw, ra)
            sb.run_frame_bytes(rgb, bw, np.ascontiguousarray(cert8), rb)
        sa.sync(); sb.sync()
        assert np.array_equal(ra, rb), i


def test_file_pipeline_and_cli_with_forward_flows(fav, tmp_path):
    """fav_video_pipeline_run_flows (via video.main -flow_pattern_forward) writes the PNGs fav_video_pipeline_run writes from the
    oracle's 4-argument PGMs, byte for byte; the Python driver with the flag gives the same pixels."""
    from PIL import Image

    from fav_b200 import video

    H, W, n = 64, 96, 5
    d = str(tmp_path)
    write_clip(d, H, W, n)
    common = ["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo", "-num_frames", str(n)]
    assert video.main(common + ["-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-output_prefix", f"{d}/pgm"])["frames"] == n
    assert video.main(common + ["-flow_pattern_forward", f"{d}/forward_{{%d}}_[%d].flo", "-output_prefix", f"{d}/flo"])["frames"] == n
    video.main(common + ["-flow_pattern_forward", f"{d}/forward_{{%d}}_[%d].flo", "-output_prefix", f"{d}/drv", "-pipeline", "0"])
    video.flush_saves()
    for i in range(1, n + 1):
        a = open(f"{d}/pgm-{i:05d}.png", "rb").read()
        assert a == open(f"{d}/flo-{i:05d}.png", "rb").read(), i
        assert np.array_equal(np.asarray(Image.open(f"{d}/drv-{i:05d}.png")), np.asarray(Image.open(f"{d}/pgm-{i:05d}.png"))), i
