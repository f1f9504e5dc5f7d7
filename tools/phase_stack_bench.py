#!/usr/bin/env python
"""phase_stack_bench.py -- stacked sub-pixel phases: run_next_image of the default arch at 1280x720 planned with one job per
sub-pixel phase of u64 and u32 (FAV_NO_STACK=1) and with the phases stacked along N, the same seeded weights; one JSON line on
stdout.

  python tools/phase_stack_bench.py --steps 300 --warmup 20 --repeats 3

ms per frame from CUDA events over --steps recurrent frames, the two plans alternated --repeats times in one process (min and
max reported).  The per-layer split comes from fav_net_profile (per-step CUDA events on one forward; the median of --profiles
forwards per step), also alternated --repeats times: every layer's time in both plans, and u64 + u32 summed.  Card name and
power limit are read in the same run.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from nl_bench import layer_split  # noqa: E402
from wide_bench import frame_inputs, time_frames  # noqa: E402

H, W = 720, 1280
UP = ("conv:l8", "conv:l9")  # u64, u32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profiles", type=int, default=9)
    args = ap.parse_args()
    from fav_b200 import models_video, synth
    from oracle import pyoracle

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    arch = synth.DEFAULT_ARCH
    inp = frame_inputs(H, W, dev)
    x7 = torch.from_numpy(pyoracle.first_frame_input(synth.make_frame(H, W, 1)).astype(np.float32))[None].to(dev)
    nets = {}
    for name in ("per_phase", "stacked"):  # the plan (and FAV_NO_STACK) is fixed at a net's first call at a size
        os.environ.pop("FAV_NO_STACK", None)
        if name == "per_phase":
            os.environ["FAV_NO_STACK"] = "1"
        nets[name] = models_video.synthetic_model("candy", arch)
        time_frames(nets[name], inp, args.warmup)
        nets[name].profile(x7)
    os.environ.pop("FAV_NO_STACK", None)
    times = {n: [] for n in nets}
    splits = {n: [] for n in nets}
    for _ in range(args.repeats):  # alternated: a drifting clock affects both alike
        for n in nets:
            times[n].append(time_frames(nets[n], inp, args.steps))
        for n in nets:
            splits[n].append(layer_split(nets[n], x7, args.profiles))
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    res, layers = {}, {}
    for n, t in times.items():
        up = [sum(s[k] for k in UP) for s in splits[n]]
        res[n] = {"ms_per_frame": round(min(t), 4), "ms_per_frame_max": round(max(t), 4),
                  "u64_u32_ms": round(min(up), 4), "u64_u32_ms_max": round(max(up), 4),
                  "u64_ms": [s[UP[0]] for s in splits[n]], "u32_ms": [s[UP[1]] for s in splits[n]]}
    for k in splits["per_phase"][0]:
        layers[k] = {n: [s.get(k) for s in splits[n]] for n in nets}
    print(json.dumps({"metric": "phase_stack_ms_per_frame", "arch": arch, "frame": [H, W], "gpu": gpu, "steps": args.steps,
                      "repeats": args.repeats, "results": res,
                      "speedup": round(res["per_phase"]["ms_per_frame"] / res["stacked"]["ms_per_frame"], 4),
                      "layers": layers}), flush=True)


if __name__ == "__main__":
    main()
