"""Single-pass fp16 mode against the exact pair mode (fav_net_set_precision), in one process, the two modes alternating, three
repeats: ms per frame (run_image, CUDA graph) at 1280x720, 1920x1080, 3840x2160 and a 2048x2048 face, aggregate frames/s of a
256x256 batch of 8, per-conv ms (fav_net_profile, 720p), max-abs against the exact mode and against the fp64 oracle at 720p, and
fav_temporal_mse of a 30-frame clip in each mode.  Prints the card and its power limit, read in the same run, and one JSON line.
    python tools/precision_bench.py [--out results/precision_bench.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fast-artistic-videos_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from fav_b200 import models_video, synth  # noqa: E402

MODES = ("pair", "fp16")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def time_frames(net, H, W, B=1, iters=20):
    x = torch.from_numpy(np.stack([synth.make_frame(H, W, 1 + b) for b in range(B)])).cuda()
    run = (lambda: net.run_image(x[0])) if B == 1 else (lambda: net.forward(torch.cat([x, x[:, :1].repeat(1, 4, 1, 1)], 1)))
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def clip_frames(net, H, W, n=30):
    from fav_b200 import consistencyChecker, utils
    outs, prev = [], None
    for i in range(1, n + 1):
        f = torch.from_numpy(synth.make_frame(H, W, i)).cuda()
        if i == 1:
            prev = net.run_image(f)
        else:
            bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
            _, cert = consistencyChecker.check(torch.from_numpy(bw).cuda(), torch.from_numpy(fw).cuda(), want_cert=True)
            prev = net.run_next_image(f, prev, torch.from_numpy(synth.checker_to_lua(bw)).cuda(), utils.min_filter(cert, 7))
        outs.append(prev.clone())
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    nets = {m: models_video.synthetic_model("candy") for m in MODES}
    nets["fp16"].set_precision("fp16")
    res = {"card": card(), "repeats": a.repeats, "ms_per_frame": {}, "batch8_256_fps": {}}
    sizes = [(720, 1280), (1080, 1920), (2160, 3840), (2048, 2048)]
    for H, W in sizes:
        key = f"{W}x{H}"
        res["ms_per_frame"][key] = {m: [] for m in MODES}
        for r in range(a.repeats):
            for m in MODES:
                res["ms_per_frame"][key][m].append(round(time_frames(nets[m], H, W), 4))
    res["batch8_256_fps"] = {m: [] for m in MODES}
    for r in range(a.repeats):
        for m in MODES:
            ms = time_frames(nets[m], 256, 256, B=8)
            res["batch8_256_fps"][m].append(round(8000.0 / ms, 1))
    # per-conv device time, 720p (fav_net_profile: CUDA events around every plan step)
    x7 = torch.cat([torch.from_numpy(synth.make_frame(720, 1280, 1))] * 2 + [torch.zeros(1, 720, 1280)]).cuda()[None]
    res["per_conv_ms_720p"] = {}
    for m in MODES:
        nets[m].profile(x7)
        per = {}
        for r in range(a.repeats):
            for s_ in nets[m].profile(x7):
                if s_["kind"] == "conv":
                    per.setdefault(s_["name"], []).append(s_["ms"])
        res["per_conv_ms_720p"][m] = {k: round(min(v), 4) for k, v in per.items()}
    # accuracy at 720p
    from oracle import net_oracle
    f = synth.make_frame(720, 1280, 1)
    ft = torch.from_numpy(f).cuda()
    o = {m: nets[m].run_image(ft).cpu().numpy() for m in MODES}
    ref = net_oracle.NetOracle(style="candy", dtype=torch.float64).run_image(f)
    res["maxabs_720p"] = {"fp16_vs_pair": float(np.abs(o["fp16"] - o["pair"]).max()),
                          "fp16_vs_fp64": float(np.abs(o["fp16"] - ref).max()),
                          "pair_vs_fp64": float(np.abs(o["pair"] - ref).max())}
    # temporal consistency of a 30-frame 256x256 clip (fav_temporal_mse between consecutive outputs), and the drift between
    # the modes (max-abs every fifth frame)
    from fav_b200 import consistencyChecker, utils
    clips = {m: clip_frames(nets[m], 256, 256) for m in MODES}
    res["clip30_256_drift_maxabs"] = [round(float((p_ - q_).abs().max()), 5) for p_, q_ in zip(clips["pair"], clips["fp16"])][::5]
    res["temporal_mse_clip30"] = {}
    for m in MODES:
        tot = 0.0
        for i in range(2, 31):
            bw, fw = synth.make_backward_flow(256, 256, i), synth.make_forward_flow(256, 256, i)
            _, cert = consistencyChecker.check(torch.from_numpy(bw).cuda(), torch.from_numpy(fw).cuda(), want_cert=True)
            tot += utils.temporal_loss(clips[m][i - 2], clips[m][i - 1], torch.from_numpy(synth.checker_to_lua(bw)).cuda(), cert)
        res["temporal_mse_clip30"][m] = tot / 29
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
