#!/usr/bin/env python
"""wide_bench.py -- run_next_image of the default arch and of the same arch at twice the width (256-channel residual blocks,
run as two 128-channel N-block jobs per convolution) at 1280x720 and at a 2048x2048 VR cube face; one JSON line on stdout.

  python tools/wide_bench.py --steps 50 --warmup 5 --repeats 3

ms per frame from CUDA events over --steps recurrent frames, the configurations alternated --repeats times in one process
(min and max reported).  Algorithmic conv FLOPs use logical channels (2 Cin Cout k^2 per output pixel, as bench.py counts
them); TFLOP/s are over the conv kernels' time from fav_net_profile (per-step CUDA events on one forward), overall and for
the residual convolutions alone, plus the profile's per-layer split in ms.  Seeded weights (synth.make_weights).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "fast-artistic-videos_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

ARCHS = {"default": "c9s1-32,d64,d128,R128,R128,R128,R128,R128,u64,u32,c9s1-3",
         "doubled": "c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3"}
SIZES = {"720p": (720, 1280), "vr_face_2048": (2048, 2048)}


def frame_inputs(H, W, dev):
    from fav_b200 import synth
    from oracle import net_oracle

    frame = torch.from_numpy(synth.make_frame(H, W, 2)).to(dev)
    prev = torch.from_numpy(synth.make_frame(H, W, 1)).to(dev)
    flow = torch.from_numpy(synth.checker_to_lua(synth.make_backward_flow(H, W, 2))).to(dev)
    cert = torch.from_numpy(net_oracle.make_cert(H, W, 2)).to(dev)
    return frame, prev, flow, cert


def time_frames(net, inp, steps):
    frame, prev, flow, cert = inp
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        prev = net.run_next_image(frame, prev, flow, cert)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def profile(net, H, W, dev):
    from fav_b200 import synth
    from oracle import pyoracle

    x7 = torch.from_numpy(pyoracle.first_frame_input(synth.make_frame(H, W, 1)).astype(np.float32))[None].to(dev)
    net.profile(x7)  # warm-up; the second profiled forward is the one reported
    steps = net.profile(x7)
    conv = [s for s in steps if s["kind"] == "conv"]
    res = [s for s in conv if ".c" in s["name"]]
    tf = lambda ss: round(sum(s["work"] for s in ss) / (sum(s["ms"] for s in ss) * 1e-3) / 1e12, 1)
    return {"conv_gflop": round(sum(s["work"] for s in conv) / 1e9, 1),
            "conv_ms": round(sum(s["ms"] for s in conv), 3), "conv_tflops": tf(conv),
            "residual_conv_ms": round(sum(s["ms"] for s in res), 3), "residual_conv_tflops": tf(res),
            "layers_ms": {f"{s['kind']}:{s['name']}": round(s["ms"], 4) for s in steps}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from fav_b200 import models_video

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    nets = {a: models_video.synthetic_model("candy", arch) for a, arch in ARCHS.items()}
    inputs = {s: frame_inputs(H, W, dev) for s, (H, W) in SIZES.items()}
    configs = [(a, s) for s in SIZES for a in ARCHS]
    for a, s in configs:
        time_frames(nets[a], inputs[s], args.warmup)
    times = {c: [] for c in configs}
    for _ in range(args.repeats):  # the configurations alternate: a drifting clock affects all of them alike
        for c in configs:
            times[c].append(time_frames(nets[c[0]], inputs[c[1]], args.steps))
    results = {}
    for a, s in configs:
        H, W = SIZES[s]
        prof = profile(nets[a], H, W, dev)
        ms = min(times[(a, s)])
        results[f"{a}@{s}"] = {"arch": ARCHS[a], "frame": [H, W], "ms_per_frame": round(ms, 3),
                               "ms_per_frame_max": round(max(times[(a, s)]), 3),
                               "conv_tflops_algorithmic_over_frame_time": round(prof["conv_gflop"] * 1e9 / (ms * 1e-3) / 1e12, 1),
                               **prof}
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    print(json.dumps({"metric": "wide_net_ms_per_frame", "gpu": gpu, "steps": args.steps, "repeats": args.repeats,
                      "results": results}), flush=True)


if __name__ == "__main__":
    main()
