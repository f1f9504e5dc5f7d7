#!/usr/bin/env python
"""style_bank_bench.py -- B clips in B styles advancing one frame per call, default arch, at 256x256, 640x360 and 1280x720 with
B in {1, 2, 4, 8}; one JSON line on stdout.

  python tools/style_bank_bench.py --steps 30 --warmup 3 --repeats 3

Three legs per configuration, alternated --repeats times in one process (best and worst reported):
  bank:     one net holding B styles (fav_net_add_style), one batched run_next_image call per frame, image b in style b;
  separate: the same B clips on B separate nets, one single-frame call each per frame;
  same:     a same-style batch of B on one net (the batching this project had before style banks).
ms per frame step from CUDA events over --steps recurrent steps; aggregate frames/s = B / ms.  The bank and the separate nets
must give the same frames bit for bit (checked once per configuration).  The card's name, power limit and SM clock are read in
the same run.
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

SIZES = {"256x256": (256, 256), "640x360": (360, 640), "1280x720": (720, 1280)}
BATCHES = (1, 2, 4, 8)
STYLE_NAMES = ("candy", "mosaic", "udnie", "scream", "wave", "feathers", "muse", "composition")


def batch_inputs(H, W, B, dev):
    from fav_b200 import synth
    from oracle import net_oracle

    frame = np.stack([synth.make_frame(H, W, 2 + b) for b in range(B)])
    prev = np.stack([synth.make_frame(H, W, 1 + b) for b in range(B)])
    flow = np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 2 + b)) for b in range(B)])
    cert = np.stack([net_oracle.make_cert(H, W, 2 + b) for b in range(B)])
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (frame, prev, flow, cert)]


def step_bank(bank, inp, prev, B):
    frame, _, flow, cert = inp
    return bank.run_next_image(frame, prev, flow, cert, styles=list(range(B)))


def step_separate(nets, inp, prev, B):
    frame, _, flow, cert = inp
    return torch.stack([nets[b].run_next_image(frame[b], prev[b], flow[b], cert[b]) for b in range(B)])


def step_same(net, inp, prev, B):
    frame, _, flow, cert = inp
    return net.run_next_image(frame, prev, flow, cert)


def time_leg(step, inp, steps):
    prev = inp[1]
    B = prev.size(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        prev = step(inp, prev, B)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from fav_b200 import models_video

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    nets = [models_video.synthetic_model(s) for s in STYLE_NAMES[:max(BATCHES)]]
    banks = {}
    for B in BATCHES:  # a bank of B styles per batch size: the bank leg carries exactly the styles it runs
        banks[B] = models_video.synthetic_model(STYLE_NAMES[0])
        for s in range(1, B):
            banks[B].add_style(nets[s])
    legs = {
        "bank": lambda B: (lambda inp, prev, b: step_bank(banks[B], inp, prev, b)),
        "separate": lambda B: (lambda inp, prev, b: step_separate(nets, inp, prev, b)),
        "same": lambda B: (lambda inp, prev, b: step_same(nets[0], inp, prev, b)),
    }
    configs, inputs, identical = [], {}, {}
    for s, (H, W) in SIZES.items():
        for B in BATCHES:
            inputs[(s, B)] = inp = batch_inputs(H, W, B, dev)
            a = step_bank(banks[B], inp, inp[1], B)
            b = step_separate(nets, inp, inp[1], B)
            identical[f"B{B}@{s}"] = bool(torch.equal(a, b))
            for leg in legs:
                time_leg(legs[leg](B), inp, args.warmup)
            configs.append((s, B))
    times = {(c, leg): [] for c in configs for leg in legs}
    for _ in range(args.repeats):  # configurations and legs alternate: a drifting clock affects all of them alike
        for c in configs:
            for leg in legs:
                times[(c, leg)].append(time_leg(legs[leg](c[1]), inputs[c], args.steps))
    results = {}
    for s, B in configs:
        r = {"frame": list(SIZES[s]), "B": B, "bit_identical_to_separate_nets": identical[f"B{B}@{s}"]}
        for leg in legs:
            t = times[((s, B), leg)]
            r[leg] = {"ms_per_step": round(min(t), 3), "ms_per_step_max": round(max(t), 3),
                      "frames_per_s": round(B * 1e3 / min(t), 1), "frames_per_s_min": round(B * 1e3 / max(t), 1)}
        r["bank_vs_separate"] = round(r["bank"]["frames_per_s"] / r["separate"]["frames_per_s"], 3)
        r["bank_vs_same"] = round(r["bank"]["frames_per_s"] / r["same"]["frames_per_s"], 3)
        results[f"B{B}@{s}"] = r
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = torch.cuda.get_device_name(0)
    print(json.dumps({"metric": "style_bank_frames_per_s", "gpu": gpu, "steps": args.steps, "repeats": args.repeats,
                      "results": results}), flush=True)


if __name__ == "__main__":
    main()
