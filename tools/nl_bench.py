#!/usr/bin/env python
"""nl_bench.py -- norm-on-load: run_next_image of the default arch at 1280x720 planned with every InstanceNorm pass separate
(FAV_NO_NL=1) and with the passes folded into the convolutions that read them, the same seeded weights; one JSON line on stdout.

  python tools/nl_bench.py --steps 300 --warmup 20 --repeats 3

ms per frame from CUDA events over --steps recurrent frames, the two plans alternated --repeats times in one process (min and
max reported).  The per-layer split comes from fav_net_profile (per-step CUDA events on one forward; the median of --profiles
forwards per step): each consumer conv's time in both plans, and the in_apply passes only the separate plan runs.  Card name
and power limit are read in the same run.
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

from wide_bench import frame_inputs, time_frames  # noqa: E402

H, W = 720, 1280


def layer_split(net, x7, n):
    runs = [net.profile(x7) for _ in range(n + 1)][1:]  # the first profiled forward is a warm-up
    out = {}
    for i, s in enumerate(runs[0]):
        out[f"{s['kind']}:{s['name']}"] = round(float(np.median([r[i]["ms"] for r in runs])), 4)
    return out


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
    nets = {}
    for name in ("separate", "fused"):  # the plan (and FAV_NO_NL) is fixed at a net's first frame of a size
        os.environ.pop("FAV_NO_NL", None)
        if name == "separate":
            os.environ["FAV_NO_NL"] = "1"
        nets[name] = models_video.synthetic_model("candy", arch)
        time_frames(nets[name], inp, args.warmup)
    os.environ.pop("FAV_NO_NL", None)
    times = {n: [] for n in nets}
    for _ in range(args.repeats):  # alternated: a drifting clock affects both alike
        for n in nets:
            times[n].append(time_frames(nets[n], inp, args.steps))
    x7 = torch.from_numpy(pyoracle.first_frame_input(synth.make_frame(H, W, 1)).astype(np.float32))[None].to(dev)
    split = {n: layer_split(nets[n], x7, args.profiles) for n in nets}
    layers = {}
    for k in split["separate"]:
        layers[k] = {"separate_ms": split["separate"][k], "fused_ms": split["fused"].get(k)}
    folded = [k for k in split["separate"] if k not in split["fused"]]
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    res = {n: {"ms_per_frame": round(min(t), 4), "ms_per_frame_max": round(max(t), 4),
               "profile_sum_ms": round(sum(split[n].values()), 4)} for n, t in times.items()}
    print(json.dumps({"metric": "norm_on_load_ms_per_frame", "arch": arch, "frame": [H, W], "gpu": gpu, "steps": args.steps,
                      "repeats": args.repeats, "results": res,
                      "speedup": round(res["separate"]["ms_per_frame"] / res["fused"]["ms_per_frame"], 4),
                      "folded_passes": folded, "layers": layers}), flush=True)


if __name__ == "__main__":
    main()
