#!/usr/bin/env python
"""batch_bench.py -- B independent clips advancing one frame per batched run_next_image call (fav_run_next_image_batch), default
arch, at 256x256, 640x360, 1280x720 and 1920x1080 with B in {1, 2, 4, 8}; one JSON line on stdout.

  python tools/batch_bench.py --steps 30 --warmup 3 --repeats 3

Per configuration: ms per batched call from CUDA events over --steps recurrent calls (the configurations alternated --repeats
times in one process; min and max reported), aggregate frames/s = B / ms, and -- in a separate run under torch.profiler -- the
device time of the conv_tc_kernel launches of one batched forward (ms per batch and per frame).  The card's name and power
limit are read in the same run.  A configuration whose activations exceed the per-plan cap (include/fav.h) is reported as
refused.
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

SIZES = {"256x256": (256, 256), "640x360": (360, 640), "1280x720": (720, 1280), "1920x1080": (1080, 1920)}
BATCHES = (1, 2, 4, 8)


def batch_inputs(H, W, B, dev):
    from fav_b200 import synth
    from oracle import net_oracle

    frame = np.stack([synth.make_frame(H, W, 2 + b) for b in range(B)])
    prev = np.stack([synth.make_frame(H, W, 1 + b) for b in range(B)])
    flow = np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 2 + b)) for b in range(B)])
    cert = np.stack([net_oracle.make_cert(H, W, 2 + b) for b in range(B)])
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (frame, prev, flow, cert)]


def time_calls(net, inp, steps):
    frame, prev, flow, cert = inp
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        prev = net.run_next_image(frame, prev, flow, cert)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def conv_kernel_ms(net, H, W, B, dev):
    """Device time of the conv_tc_kernel launches of one batched forward (eager launches, torch.profiler / CUPTI)."""
    from torch.profiler import ProfilerActivity, profile

    x = torch.rand((B, 7, H, W), device=dev) * 100
    net.forward(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net.forward(x)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "conv_tc_kernel" in e.key)
    return us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from fav_b200 import _lib, models_video

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    net = models_video.synthetic_model("candy")
    configs, inputs, refused = [], {}, {}
    for s, (H, W) in SIZES.items():
        for B in BATCHES:
            try:
                inputs[(s, B)] = batch_inputs(H, W, B, dev)
                time_calls(net, inputs[(s, B)], args.warmup)
                configs.append((s, B))
            except _lib.FavError as e:
                refused[f"B{B}@{s}"] = e.message
                inputs.pop((s, B), None)
    times = {c: [] for c in configs}
    for _ in range(args.repeats):  # the configurations alternate: a drifting clock affects all of them alike
        for c in configs:
            times[c].append(time_calls(net, inputs[c], args.steps))
    results = {}
    for s, B in configs:
        H, W = SIZES[s]
        ms = min(times[(s, B)])
        conv = conv_kernel_ms(net, H, W, B, dev)
        results[f"B{B}@{s}"] = {"frame": [H, W], "B": B, "ms_per_batch": round(ms, 3), "ms_per_batch_max": round(max(times[(s, B)]), 3),
                                "frames_per_s": round(B * 1e3 / ms, 1), "frames_per_s_min": round(B * 1e3 / max(times[(s, B)]), 1),
                                "conv_kernel_ms_per_batch": round(conv, 3), "conv_kernel_ms_per_frame": round(conv / B, 3)}
    for s in SIZES:
        base = results.get(f"B1@{s}")
        for B in BATCHES[1:]:
            r = results.get(f"B{B}@{s}")
            if base and r:
                r["gain_vs_B1"] = round(r["frames_per_s"] / base["frames_per_s"], 3)
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    print(json.dumps({"metric": "batched_run_next_image_frames_per_s", "gpu": gpu, "steps": args.steps, "repeats": args.repeats,
                      "results": results, "refused": refused}), flush=True)


if __name__ == "__main__":
    main()
