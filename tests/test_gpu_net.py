"""GPU parity tests of the stylization net and the frame loop, through the C ABI, vs the fp64 PyTorch oracle and the
committed golden clip.  Bar (BASELINE.json north_star): final deprocessed output within 1e-3 max-abs; the
fp16-pair (hi/lo) tensor-core path is expected near 1e-5."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from fav_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3  # north_star tolerance on the deprocessed [0,1] output


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available()
    from fav_b200 import models_video

    return models_video.synthetic_model("candy")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rand_input(H, W, seed=0):
    from oracle import pyoracle

    rng = np.random.default_rng(seed)
    x7 = pyoracle.first_frame_input(synth.make_frame(H, W, 1))
    x7[3:6] = rng.normal(0, 50, (3, H, W))
    x7[6] = rng.uniform(0, 1, (H, W))
    return x7.astype(np.float32)


# 48x508 / 48x516: the residual convs output widths 127 ... 145 / 129 ... 147, so tiles end 1 pixel short of or 1 pixel into
# a 128-pixel tile (H stays above the reflection pad of 40)
@pytest.mark.parametrize("shape", [(64, 96), (128, 200), (256, 256), (48, 508), (48, 516)])
@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_net_forward_and_every_layer_vs_fp64_oracle(net, shape, impl):
    from oracle import net_oracle

    H, W = shape
    net.set_conv_impl(impl)
    try:
        ora = net_oracle.NetOracle(style="candy", dtype=torch.float64)
        x7 = rand_input(H, W)
        taps = {}
        ref = ora.forward(torch.from_numpy(x7)[None], taps)[0].numpy()
        out = net.forward(T(x7)[None]).cpu().numpy()[0]
        for i in range(len(ora.specs) - 1):  # every arch token's activation (post IN / ReLU / residual add)
            r = taps[f"l{i}"][0].numpy()
            g = net.layer_output(i).cpu().numpy()
            assert g.shape == r.shape
            assert np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"layer {i}"
        assert np.abs(out - ref).max() / 255.0 < TOL / 10  # net space is 255x the [0,1] output
    finally:
        net.set_conv_impl("tcgen05")


@pytest.mark.parametrize("shape", [(64, 96), (200, 256)])
def test_paper_arch_with_nearest_upsampling(shape):
    """The arch of the paper's released models: ...,U2,c3s1-64,U2,c9s1-3 (README.md:256): UX = nearest upsampling followed
    by InstanceNorm + ReLU (models_video.lua:94-98,121-130)."""
    from fav_b200 import models_video
    from oracle import net_oracle

    H, W = shape
    net_u = models_video.synthetic_model("mosaic", synth.PAPER_ARCH)
    ora = net_oracle.NetOracle(arch=synth.PAPER_ARCH, style="mosaic", dtype=torch.float64)
    x7 = rand_input(H, W, 5)
    taps = {}
    ref = ora.forward(torch.from_numpy(x7)[None], taps)[0].numpy()
    out = net_u.forward(T(x7)[None]).cpu().numpy()[0]
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = net_u.layer_output(i).cpu().numpy()
        assert g.shape == r.shape and np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"layer {i}"
    assert np.abs(out - ref).max() / 255.0 < TOL / 10
    f1 = synth.make_frame(H, W, 1)
    assert np.abs(net_u.run_image(T(f1)).cpu().numpy() - ora.run_image(f1)).max() < TOL / 10


@pytest.mark.parametrize("arch,ptype", [
    ("c9s1-32,d64,C64,R64,f3s2-32,f3s1-32,c9s1-3", "reflect-start"),   # CX block, fXsY-Z full convolutions (stride 2 and 1), 64-ch blocks
    ("c9s1-32,d64,d128,R128,R128,f5s2-64,u32,c9s1-3", "reflect-start"),  # 5x5 full convolution: 4 sub-pixel phases with 9/6/6/4 taps
    (synth.DEFAULT_ARCH, "zero"),                                       # padding_type zero: padded residual convs, Identity skip
    # wgmma N = 16 / 48 / 80, a residual block with 10 channel blocks (CbG 2, norm-on-load), x-fold from 16 channels (CbG 2)
    ("c9s1-16,d48,d80,R80,R80,u48,u16,c9s1-3", "reflect-start"),
    ("c9s1-32,d96,d112,R112,u96,u32,c5s1-3", "reflect-start"),         # N = 96 / 112; x-fold c5s1-3 with N = 5 x 3 -> 16
    ("c9s1-32,d64,d128,R128,u32,u8,c9s1-3", "reflect-start"),          # Cout 8 (N 16, padded IN statistics); final conv
                                                                       # from 8 channels: tap pairing, plain final epilogue
    ("c9s1-32,d64,R64,u32,c3s1-3", "zero"),                             # generic final conv (N = 16), plain final epilogue
])
def test_arch_tokens_and_padding_types(arch, ptype):
    """models_video.build_model's remaining tokens (fXsY-Z :81-89, CX :103-108) and padding_type 'zero' (:13-19,46-50) vs the
    fp64 oracle, every layer."""
    from fav_b200 import models_video
    from oracle import net_oracle

    H, W = 64, 96
    w = synth.make_weights(arch, "scream")
    net_x = models_video.StyleNet(arch, padding_type=ptype).load_state(w)
    ora = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype)
    x7 = rand_input(H, W, 9)
    taps = {}
    ref = ora.forward(torch.from_numpy(x7)[None], taps)[0].numpy()
    out = net_x.forward(T(x7)[None]).cpu().numpy()[0]
    assert out.shape == ref.shape == (3, H, W)
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = net_x.layer_output(i).cpu().numpy()
        assert g.shape == r.shape and np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"layer {i}"
    assert np.abs(out - ref).max() / 255.0 < TOL / 10
    f1 = synth.make_frame(H, W, 1)
    assert np.abs(net_x.run_image(T(f1)).cpu().numpy() - ora.run_image(f1)).max() < TOL / 10


def test_unsupported_padding_types_fail_loudly():
    from fav_b200 import _lib, models_video

    for ptype in ("reflect", "replicate", "none"):
        with pytest.raises(_lib.FavError) as e:
            models_video.StyleNet(synth.DEFAULT_ARCH, padding_type=ptype)
        assert e.value.status == _lib.FAV_ERR_UNSUPPORTED


def test_tcgen05_agrees_with_cuda_core_comparator(net):
    x = T(rand_input(96, 160, 3))[None]
    a = net.forward(x)
    net.set_conv_impl("simt")
    try:
        b = net.forward(x)
    finally:
        net.set_conv_impl("tcgen05")
    assert float((a - b).abs().max()) / 255.0 < 5e-5


def test_golden_clip_recurrence(net):
    """3-frame clip through run_image / run_next_image with the occlusion mask computed on the GPU, vs the committed
    fp64 oracle outputs (tests/golden/clip_64x96.npz); the recurrent state stays on the device."""
    from fav_b200 import consistencyChecker, utils

    g = np.load(os.path.join(ROOT, "tests", "golden", "clip_64x96.npz"))["outs"]
    H, W = 64, 96
    prev = None
    for i in range(1, 4):
        frame = T(synth.make_frame(H, W, i))
        if i == 1:
            out = net.run_image(frame)
        else:
            bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
            _, cert = consistencyChecker.check(T(bw), T(fw), want_cert=True)
            cert = utils.min_filter(cert, 7)
            out = net.run_next_image(frame, prev, T(synth.checker_to_lua(bw)), cert)
        err = float(np.abs(out.cpu().numpy() - g[i - 1]).max())
        assert err < TOL, (i, err)
        assert err < 1e-4, (i, err)  # what the hi/lo scheme actually delivers
        prev = out


@pytest.mark.parametrize("shape", [(256, 256), (360, 640)])
def test_run_next_image_teacher_forced(net, shape):
    from oracle import net_oracle

    H, W = shape
    ora = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    f1, f2 = synth.make_frame(H, W, 1), synth.make_frame(H, W, 2)
    ref1 = ora.run_image(f1)
    out1 = net.run_image(T(f1)).cpu().numpy()
    assert np.abs(out1 - ref1).max() < TOL / 10
    cert = net_oracle.make_cert(H, W, 2)
    flow = synth.checker_to_lua(synth.make_backward_flow(H, W, 2))
    prev = ref1.astype(np.float32)
    for border in (0, 1):  # CUDA and CPU warp semantics of utils.warp_image
        ref2 = ora.run_next_image(f2, prev, flow, cert, warp_mode=border)
        out2 = net.run_next_image(T(f2), T(prev), T(flow), T(cert), border_mode=border).cpu().numpy()
        assert np.abs(out2 - ref2).max() < TOL / 10


def test_session_host_buffer_loop_matches_device_api(net):
    """fav_session_* (pinned host buffers, 3 streams) == the device-pointer API, and the fused-flow variant
    (occlusion mask from the flow pair on the GPU) == explicit consistencyChecker + min_filter."""
    from fav_b200 import consistencyChecker, session, utils

    H, W = 96, 128
    s = session.Session(net, H, W)
    frames = [torch.from_numpy(synth.make_frame(H, W, i)).pin_memory() for i in range(1, 5)]
    outs = [torch.empty((3, H, W)).pin_memory() for _ in range(4)]
    s.run_image(frames[0], outs[0])
    for i in range(2, 5):
        bw = torch.from_numpy(synth.make_backward_flow(H, W, i)).pin_memory()
        fw = torch.from_numpy(synth.make_forward_flow(H, W, i)).pin_memory()
        s.run_next_image_flows(frames[i - 1], bw, fw, outs[i - 1], 7)
    s.sync()
    assert s.last_gpu_ms() > 0
    prev = net.run_image(frames[0].cuda())
    assert torch.equal(prev.cpu(), outs[0])
    for i in range(2, 5):
        bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
        _, cert = consistencyChecker.check(T(bw), T(fw), want_cert=True)
        prev = net.run_next_image(frames[i - 1].cuda(), prev, T(synth.checker_to_lua(bw)), utils.min_filter(cert, 7))
        assert torch.equal(prev.cpu(), outs[i - 1]), i
    # cert-given variant
    s2 = session.Session(net, H, W)
    o1, o2 = torch.empty((3, H, W)).pin_memory(), torch.empty((3, H, W)).pin_memory()
    s2.run_image(frames[0], o1)
    bw = synth.make_backward_flow(H, W, 2)
    cert_raw = consistencyChecker.check(T(bw), T(synth.make_forward_flow(H, W, 2)), want_cert=True)[1].cpu().pin_memory()
    s2.run_next_image(frames[1], torch.from_numpy(synth.checker_to_lua(bw)).pin_memory(), cert_raw, o2, 7)
    s2.sync()
    assert torch.equal(o2, outs[1])


def test_session_file_payload_path_matches_float_path(net):
    """fav_session_run_frame_bytes (P6 / P5 / .flo payloads in, Sub-filtered PNG scanlines out; byte <-> float conversions on the
    GPU) == the host-side conversions of the float path (image.load's byte/255, -invert_occlusion, image.save's rounding)."""
    from fav_b200 import session

    H, W = 96, 128
    rng = np.random.default_rng(5)
    rgb = [torch.from_numpy(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).pin_memory() for _ in range(3)]
    cert8 = [torch.from_numpy(((rng.uniform(size=(H, W)) > 0.2) * 255).astype(np.uint8)).pin_memory() for _ in range(3)]
    flo = [torch.from_numpy(np.ascontiguousarray(synth.make_backward_flow(H, W, i + 2).transpose(1, 2, 0))).pin_memory() for i in range(3)]
    for invert in (False, True):
        sb = session.Session(net, H, W)
        rows = [torch.zeros((H, 1 + 3 * W), dtype=torch.uint8).pin_memory() for _ in range(3)]
        outs = [torch.empty((3, H, W)).pin_memory() for _ in range(3)]
        for i in range(3):
            sb.run_frame_bytes(rgb[i], flo[i] if i else None, cert8[i] if i else None, rows[i], invert_occlusion=invert)
        assert sb.frame_done(2)
        sb.sync()  # one net = one set of activation buffers: the two sessions must not overlap
        sf = session.Session(net, H, W)
        keep = []
        for i in range(3):
            content = (rgb[i].permute(2, 0, 1).float() / 255.0).contiguous().pin_memory()
            keep.append(content)
            if i == 0:
                sf.run_image(content, outs[i])
            else:
                cert = cert8[i].float() / 255.0
                if invert:
                    cert = 1.0 - cert
                lua_flow = torch.stack([flo[i][..., 1], flo[i][..., 0]]).contiguous().pin_memory()  # (dy, dx), flowFileLoader.lua:31-32
                cert = cert.contiguous().pin_memory()
                keep += [lua_flow, cert]
                sf.run_next_image(content, lua_flow, cert, outs[i], 7)
        assert sf.frame_done(2)
        sf.sync()
        for i in range(3):
            q = torch.floor(outs[i].clamp(0, 1) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8).permute(1, 2, 0).reshape(H, 3 * W)  # image.save
            r = rows[i]
            assert bool((r[:, 0] == 1).all())
            sub = r[:, 1:].to(torch.int16)
            recon = torch.zeros((H, 3 * W), dtype=torch.int16)
            for x in range(W):  # undo the Sub filter (bytes, modulo 256)
                prev = recon[:, 3 * (x - 1):3 * x] if x else 0
                recon[:, 3 * x:3 * x + 3] = (sub[:, 3 * x:3 * x + 3] + prev) % 256
            assert torch.equal(recon.to(torch.uint8), q), (invert, i)


def test_full_size_720p_properties(net):
    """BASELINE.json config 2 size.  The fp64 oracle needs ~10 s per 720p frame on a few cores, so one frame is checked
    against it and the rest through properties: determinism, and invariance of frame 1 to the (masked) prior."""
    from oracle import net_oracle

    H, W = 720, 1280
    f1 = synth.make_frame(H, W, 1)
    a = net.run_image(T(f1))
    b = net.run_image(T(f1))
    assert torch.equal(a, b)  # deterministic (no atomics on the output path)
    assert torch.isfinite(a).all()
    ora = net_oracle.NetOracle(style="candy", dtype=torch.float32)
    ref = ora.run_image(f1)
    assert np.abs(a.cpu().numpy() - ref).max() < TOL / 10
    # certainty 0 everywhere => the prior must not influence the output (core.lua:167: prior * cert)
    flow = T(synth.checker_to_lua(synth.make_backward_flow(H, W, 2)))
    zc = torch.zeros((H, W), device="cuda")
    o1 = net.run_next_image(T(f1), a, flow, zc)
    o2 = net.run_next_image(T(f1), torch.rand_like(a), flow, zc)
    assert torch.equal(o1, o2) and torch.equal(o1, a)


def test_separate_image_model_for_single_images(tmp_path):
    """-model_img (fast_artistic_video.lua:24 default is an image model; core.lua:61-68,146): frame 1 = model_img(pre(img)),
    a 3-channel-input net; later frames = the video model.  C ABI, host-buffer session and the Lua-driver mirror vs the fp64
    oracle."""
    from fav_b200 import core, models_video, session
    from oracle import net_oracle

    H, W = 64, 96
    img_net = models_video.synthetic_model("mosaic", synth.DEFAULT_ARCH, in_dim=3)
    vid_net = models_video.synthetic_model("candy")
    o_img = net_oracle.NetOracle(style="mosaic", dtype=torch.float64, in_dim=3)
    o_vid = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    f1, f2 = synth.make_frame(H, W, 1), synth.make_frame(H, W, 2)
    ref1 = o_img.run_image(f1)
    out1 = img_net.run_image(T(f1))
    assert np.abs(out1.cpu().numpy() - ref1).max() < TOL / 10
    assert np.abs(out1.cpu().numpy() - o_vid.run_image(f1)).max() > 1e-2  # really a different model
    # session: frame 1 through the image model, frame 2 through the video model with frame 1 as the prior
    s = session.Session(vid_net, H, W)
    s.set_image_model(img_net)
    o1, o2 = torch.empty((3, H, W)).pin_memory(), torch.empty((3, H, W)).pin_memory()
    bw, fw = synth.make_backward_flow(H, W, 2), synth.make_forward_flow(H, W, 2)
    s.run_image(torch.from_numpy(f1).pin_memory(), o1)
    s.run_next_image_flows(torch.from_numpy(f2).pin_memory(), torch.from_numpy(bw).pin_memory(), torch.from_numpy(fw).pin_memory(), o2, 7)
    s.sync()
    assert torch.equal(o1, out1.cpu())
    ref2 = o_vid.run_next_image(f2, o1.numpy(), synth.checker_to_lua(bw), net_oracle.make_cert(H, W, 2))
    assert np.abs(o2.numpy() - ref2).max() < TOL / 10
    # the driver mirror (run_fast_neural_video with opt.model_img)
    saved = {}
    opt = dict(model_vid="synthetic:candy", model_img="synthetic:mosaic", num_frames=2, gpu=0)
    core.run_fast_neural_video(
        opt, lambda o, i, d: T(synth.make_frame(H, W, i)) if i <= 2 else None,
        lambda o, i, d: torch.from_numpy(net_oracle.make_cert(H, W, i)).cuda(), None,
        lambda o, i, d, c: core.FusedWarp(saved[i - 1], T(synth.checker_to_lua(synth.make_backward_flow(H, W, i)))),
        lambda i, o: i == 1, lambda o, i, img, d=None: saved.__setitem__(i, img.clone()))
    assert torch.equal(saved[1].cpu(), o1)


def test_error_behaviour(net):
    from fav_b200 import _lib

    with pytest.raises(_lib.FavError) as e:
        net.forward(torch.zeros((1, 7, 50, 64), device="cuda"))  # H not a multiple of 4
    assert e.value.status == _lib.FAV_ERR_INVALID
    with pytest.raises(AssertionError):
        net.forward(torch.zeros((1, 3, 64, 64), device="cuda"))


def test_video_driver_end_to_end_files(tmp_path):
    """fast_artistic_video.lua equivalent on files: PPM frames + .flo + PGM certainty (written by the GPU
    consistencyChecker CLI) -> PNGs; the recurrent state is the unclamped fp32 frame, not the PNG (fav.lua:169)."""
    from PIL import Image

    from fav_b200 import consistencyChecker, t7, video
    from oracle import net_oracle, pyoracle

    H, W, n = 64, 96, 3
    d = str(tmp_path)
    for i in range(1, n + 1):
        synth.write_ppm(f"{d}/frame_{i:04d}.ppm", synth.make_frame(H, W, i))
    for i in range(2, n + 1):
        synth.write_flo(f"{d}/backward_{i}_{i - 1}.flo", synth.make_backward_flow(H, W, i))
        synth.write_flo(f"{d}/forward_{i - 1}_{i}.flo", synth.make_forward_flow(H, W, i))
        consistencyChecker.main(["consistencyChecker", f"{d}/backward_{i}_{i - 1}.flo", f"{d}/forward_{i - 1}_{i}.flo",
                                 f"{d}/reliable_{i}_{i - 1}.pgm"])
    # weights through a Torch7 .t7 checkpoint (f-1)
    w = synth.make_weights(synth.DEFAULT_ARCH, "candy")
    t7.write_checkpoint(f"{d}/checkpoint-candy-video.t7", synth.DEFAULT_ARCH, w)
    video.main(["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo",
                "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-model_vid", f"{d}/checkpoint-candy-video.t7",
                "-output_prefix", f"{d}/out", "-num_frames", str(n), "-evaluate", "-evaluation_file", f"{d}/evaluation.txt",
                "-flow_pattern_eval", f"{d}/backward_[%d]_{{%d}}.flo", "-occlusions_pattern_eval", f"{d}/reliable_[%d]_{{%d}}.pgm"])
    # f-2: the pipelined driver (decode threads -> pinned ring -> fav_session_* -> encoder threads) writes the SAME PNGs
    res = video.main(["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo",
                      "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-model_vid", f"{d}/checkpoint-candy-video.t7",
                      "-output_prefix", f"{d}/pipe", "-num_frames", str(n)])
    assert res["frames"] == n  # native pipeline (csrc/video_pipeline.cu): PPM / PGM / .flo inputs
    opt2 = video.build_parser().parse_args(["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo",
                                            "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-model_vid", f"{d}/checkpoint-candy-video.t7",
                                            "-output_prefix", f"{d}/pyp", "-num_frames", str(n)])
    assert video.run_pipelined(opt2, depth=4, n_decode=2, n_encode=2)["frames"] == n  # Python-thread variant (any image format)
    for i in range(1, n + 1):
        ref_png = np.asarray(Image.open(f"{d}/out-{i:05d}.png"))
        assert np.array_equal(np.asarray(Image.open(f"{d}/pipe-{i:05d}.png")), ref_png), i
        assert np.array_equal(np.asarray(Image.open(f"{d}/pyp-{i:05d}.png")), ref_png), i
    # oracle on the same files (frames are 8-bit PPMs here)
    ora = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    prev = None
    prev_prev, temporal_ref = None, []
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
        if i >= 2:  # -evaluate's temporal loss (fast_artistic_video.lua:128-151) on the oracle trajectory
            cert_eval = pyoracle.consistency(bw, fw).astype(np.float32) / 255.0
            wp = pyoracle.warp_bdhw(prev_prev, synth.checker_to_lua(bw))
            temporal_ref.append(float(np.mean(((wp - ref.astype(np.float32)) * cert_eval[None]).astype(np.float64) ** 2)))
        prev_prev = ref.astype(np.float32)
    rows = open(f"{d}/evaluation.txt").read().strip().split("\n")
    assert len(rows) == 6  # style; content; temporal per frame, then the three averages (core.lua:231-238)
    temporal = [float(v) for v in rows[2].split(";")]
    assert len(temporal) == n and temporal[0] == 0.0
    for got, want in zip(temporal[1:], temporal_ref):
        assert abs(got - want) <= 1e-6 + 1e-2 * want, (got, want)  # GPU trajectory vs oracle trajectory (1e-5 apart)
    assert abs(float(rows[5]) - sum(temporal) / n) < 1e-9
