#!/usr/bin/env python
"""percep_bench.py -- -evaluate's content and style losses for one 1280x720 frame (fast_artistic_video_core.lua:101-106) on the
GPU, one JSON line on stdout.

  python tools/percep_bench.py --steps 50 --warmup 5

Workload: VGG-16 with seeded weights in the real shapes (no network here to fetch models/vgg16.t7), the reference's default
layers: the content-target forward to relu3_3 (-content_layers 16), the stylized forward to relu4_3 (-style_layers
4,9,16,23), four Gram matrices and the losses.  ms per evaluated frame from CUDA events over --steps evaluations; the split
into convolution / Gram / other kernels from torch.profiler over a few further evaluations after the timed region.
Algorithmic FLOPs are computed from the shapes below (2 Cin Cout k^2 per output pixel; 2 C^2 H W per Gram matrix).
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

import torch  # noqa: E402

H, W = 720, 1280


def percep_flops(modules, h, w, last):
    """Algorithmic FLOPs of the loss network's convolutions up to module `last` (2 * Cin * Cout * k^2 per output pixel) at an
    h x w input, and the (h, w) of every module's output."""
    import math

    total, sizes = 0.0, {}
    for i, m in enumerate(modules[:last], 1):
        if m["type"] == "conv":
            h = (h + 2 * m["pad"] - m["k"]) // m["stride"] + 1
            w = (w + 2 * m["pad"] - m["k"]) // m["stride"] + 1
            total += 2.0 * m["cin"] * m["cout"] * m["k"] ** 2 * h * w
        elif m["type"] == "pool":
            rnd = math.ceil if m["ceil_mode"] else math.floor
            h = int(rnd((h + 2 * m["padH"] - m["kH"]) / m["dH"])) + 1
            w = int(rnd((w + 2 * m["padW"] - m["kW"]) / m["dW"])) + 1
        sizes[i] = (h, w)
    return total, sizes


def run_perceptual(args):
    """-evaluate's perceptual losses for one 720p frame (fast_artistic_video_core.lua:101-106): the content-target forward (VGG-16
    to relu3_3, the default -content_layers 16), the stylized forward (to relu4_3, -style_layers 4,9,16,23), four Gram matrices
    and the losses; seeded weights in VGG-16's shapes.  ms per evaluated frame from CUDA events; the Gram kernel's time from
    torch.profiler in a separate run."""
    from fav_b200 import percep, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    mods = percep.vgg16_modules(0)
    content_layers, style_layers = [16], [4, 9, 16, 23]
    crit = percep.PerceptualCriterion(mods, content_layers, [1.0], style_layers, [1.0] * len(style_layers))
    crit.set_style_target(torch.from_numpy(synth.make_frame(256, 256, 99)).to(dev))
    content = torch.from_numpy(synth.make_frame(H, W, 1)).to(dev)
    stylized = (content * 0.8 + 0.1).contiguous()
    for _ in range(args.warmup):
        crit.evaluate(content, stylized)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        crit.evaluate(content, stylized)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    conv_c, _ = percep_flops(mods, H, W, max(content_layers))
    conv_s, sizes = percep_flops(mods, H, W, max(content_layers + style_layers))
    chans = {i: [m for m in mods[:i] if m["type"] == "conv"][-1]["cout"] for i in style_layers}
    gram_flops = sum(2.0 * chans[i] ** 2 * sizes[i][0] * sizes[i][1] for i in style_layers)
    from torch.profiler import ProfilerActivity, profile

    reps = min(10, args.steps)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            crit.evaluate(content, stylized)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            key = "gram" if "percep_gram_kernel" in ev.name else ("conv" if "conv_tc_kernel" in ev.name else "other")
            kern[key] = kern.get(key, 0.0) + ev.device_time_total / 1e3 / reps
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    line = {"metric": "perceptual_eval_ms_per_frame", "value": round(ms, 3), "unit": "ms",
            "frame": [H, W], "steps": args.steps, "gpu": gpu,
            "conv_gflop_per_frame": round((conv_c + conv_s) / 1e9, 1), "gram_gflop_per_frame": round(gram_flops / 1e9, 1),
            "conv_tflops_algorithmic_over_frame_time": round((conv_c + conv_s) / (ms * 1e-3) / 1e12, 1),
            "profiled_ms_per_frame": {k: round(v, 3) for k, v in kern.items()},
            "conv_tflops_over_conv_kernel_time": round((conv_c + conv_s) / (kern.get("conv", float("nan")) * 1e-3) / 1e12, 1),
            "gram_tflops_over_gram_kernel_time": round(gram_flops / (kern.get("gram", float("nan")) * 1e-3) / 1e12, 1),
            "workload": "one evaluated 1280x720 frame: VGG-16 (seeded weights) content target to layer 16 + stylized to layer 23, "
                        "Gram style loss at 4,9,16,23, content loss at 16"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    run_perceptual(ap.parse_args())


if __name__ == "__main__":
    main()
