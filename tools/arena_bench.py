#!/usr/bin/env python
"""arena_bench.py -- the cost of sharing activation buffers (include/fav.h fav_net_set_activation_budget); one JSON line.

  python tools/arena_bench.py --steps 10 --warmup 2 --repeats 3

Default arch, run_image (one graph launch per frame):
  - 3840x2160: ms per frame of the all-live plan and of the arena plan (budget one byte below the all-live total), the two
    nets alternated --repeats times in one process (min and max reported): the arena plan adds one border clear per operand;
  - 7680x4320 at the default budget (an arena plan): ms per frame;
  - a batch of four 3840x2160 frames at the default budget: frames/s;
  - the planner's bytes (all-live and shared) of each plan, and the card's name and power limit, read in the same run.
Times are CUDA events around --steps calls after --warmup calls.
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


def ms_per_call(net, img, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        net.run_image(img)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from fav_b200 import models_video

    torch.cuda.set_device(0)
    gb = lambda b: round(b / 2**30, 3)  # noqa: E731
    res = {"metric": "activation_arena", "steps": args.steps, "repeats": args.repeats}

    H, W = 2160, 3840
    live = models_video.synthetic_model("candy")
    arena = models_video.synthetic_model("candy")
    all_live, shared = arena.plan_bytes(H, W)
    arena.set_activation_budget(all_live - 1)
    img = torch.rand((3, H, W), device="cuda")
    for net in (live, arena):
        ms_per_call(net, img, args.warmup)
    t = {"all_live": [], "arena": []}
    for _ in range(args.repeats):
        t["all_live"].append(ms_per_call(live, img, args.steps))
        t["arena"].append(ms_per_call(arena, img, args.steps))
    res["4k"] = {"all_live_gib": gb(all_live), "arena_gib": gb(shared),
                 "all_live_ms": [round(min(t["all_live"]), 3), round(max(t["all_live"]), 3)],
                 "arena_ms": [round(min(t["arena"]), 3), round(max(t["arena"]), 3)]}
    del live, arena, img
    torch.cuda.empty_cache()

    net = models_video.synthetic_model("candy")
    H, W = 4320, 7680
    all_live, shared = net.plan_bytes(H, W)
    img = torch.rand((3, H, W), device="cuda")
    ms_per_call(net, img, args.warmup)
    ms = [ms_per_call(net, img, args.steps) for _ in range(args.repeats)]
    res["8k"] = {"all_live_gib": gb(all_live), "arena_gib": gb(shared), "ms": [round(min(ms), 3), round(max(ms), 3)]}
    del net, img
    torch.cuda.empty_cache()

    net = models_video.synthetic_model("candy")
    B, H, W = 4, 2160, 3840
    all_live, shared = net.plan_bytes(H, W, B)
    img = torch.rand((B, 3, H, W), device="cuda")
    ms_per_call(net, img, args.warmup)
    ms = [ms_per_call(net, img, args.steps) for _ in range(args.repeats)]
    res["4k_batch4"] = {"all_live_gib": gb(all_live), "arena_gib": gb(shared),
                        "frames_per_s": [round(B * 1e3 / max(ms), 2), round(B * 1e3 / min(ms), 2)]}

    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res["gpu"] = q.stdout.strip() or torch.cuda.get_device_name(0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
