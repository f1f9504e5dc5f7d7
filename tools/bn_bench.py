#!/usr/bin/env python
"""bn_bench.py -- run_next_image of the default arch with InstanceNorm and with (inference-mode) BatchNorm, the same seeded conv
weights, at 1280x720 and at a 2048x2048 VR cube face; one JSON line on stdout.

  python tools/bn_bench.py --steps 50 --warmup 5 --repeats 3

A BN net folds each BatchNorm into its convolution and every non-final conv_tc_kernel job writes the next fp16 hi/lo operand
from its accumulators, so it has no raw fp32 store / re-read, no in_apply pass and no statistics.  ms per frame from CUDA events
over --steps recurrent frames, the configurations alternated --repeats times in one process (min and max reported).  Conv
TFLOP/s use algorithmic FLOPs (2 Cin Cout k^2 per output pixel, logical channels) over the conv kernels' time from
fav_net_profile (per-step CUDA events on one forward), plus the profile's per-layer split in ms.  BN running statistics are
calibrated on a seeded frame (tests/bn_oracle.py); the timings do not depend on them.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "fast-artistic-videos_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from wide_bench import SIZES, frame_inputs, time_frames  # noqa: E402


def profile(net, H, W, dev):
    from wide_bench import profile as wide_profile

    p = wide_profile(net, H, W, dev)
    p.pop("residual_conv_ms"), p.pop("residual_conv_tflops")
    other = sum(v for k, v in p["layers_ms"].items() if not k.startswith("conv:"))
    p["non_conv_ms"] = round(other, 3)
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import bn_oracle
    from fav_b200 import models_video, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    arch = synth.DEFAULT_ARCH
    nets = {"instance": models_video.synthetic_model("candy", arch),
            "batch": models_video.StyleNet(arch, norm="batch").load_state(bn_oracle.calibrate_bn_weights(arch, "candy"))}
    inputs = {s: frame_inputs(H, W, dev) for s, (H, W) in SIZES.items()}
    configs = [(n, s) for s in SIZES for n in nets]
    for n, s in configs:
        time_frames(nets[n], inputs[s], args.warmup)
    times = {c: [] for c in configs}
    for _ in range(args.repeats):  # the configurations alternate: a drifting clock affects all of them alike
        for c in configs:
            times[c].append(time_frames(nets[c[0]], inputs[c[1]], args.steps))
    results = {}
    for n, s in configs:
        H, W = SIZES[s]
        prof = profile(nets[n], H, W, dev)
        ms = min(times[(n, s)])
        results[f"{n}@{s}"] = {"norm": n, "frame": [H, W], "ms_per_frame": round(ms, 3), "ms_per_frame_max": round(max(times[(n, s)]), 3),
                               "conv_tflops_algorithmic_over_frame_time": round(prof["conv_gflop"] * 1e9 / (ms * 1e-3) / 1e12, 1),
                               **prof}
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    print(json.dumps({"metric": "bn_vs_in_ms_per_frame", "arch": arch, "gpu": gpu, "steps": args.steps, "repeats": args.repeats,
                      "results": results}), flush=True)


if __name__ == "__main__":
    main()
