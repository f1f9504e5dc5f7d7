#!/usr/bin/env python
"""percep_grad_bench.py -- the loss side of a training step on the GPU: PerceptualCriterion forward + backward through the
loss network (fav_percep_forward_backward), one JSON line on stdout.

  python tools/percep_grad_bench.py --steps 20 --warmup 3

Workload: VGG-16 with seeded weights in the real shapes, the reference's default layers (-content_layers 16, -style_layers
4,9,16,23, gram), at 256x256 x 4 images (train_video.lua's training shape; one call per image) and at 1280x720.  ms per
forward + backward from CUDA events over --steps calls; the split into forward convolutions, input-gradient convolutions,
Gram backward and everything else from torch.profiler over a few further calls.  The input-gradient convolutions' algorithmic
FLOPs are those of the forward convolutions they mirror (2 Cin Cout k^2 per pixel).  The card and its power limit are read in
the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "fast-artistic-videos_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CONTENT, STYLE, STYLE_W = [16], [4, 9, 16, 23], [1.0, 1.0, 1.0, 1.0]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def measure(crit, mods, H, W, nimg, steps, warmup):
    from percep_bench import percep_flops
    from fav_b200 import synth

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    mean = torch.tensor([103.939, 116.779, 123.68], device=dev)[:, None, None]
    imgs = []
    for i in range(nimg):
        c = torch.from_numpy(synth.make_frame(H, W, i + 1)).to(dev)
        s = (0.7 * c + 0.3 * torch.from_numpy(rng.uniform(-0.2, 1.2, c.shape).astype(np.float32)).to(dev))
        imgs.append(tuple((t[[2, 1, 0]] * 255.0 - mean).contiguous() for t in (c, s)))
    x = torch.stack([s for _, s in imgs])
    target = {"content_target": torch.stack([c for c, _ in imgs])}

    def step():
        crit.forward(x, target)

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    # profiler: kernel times of a few calls; the conv launches after the first backward kernel are input gradients
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
    evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0],
                 key=lambda e: e.time_range.start)
    split = {"fwd_conv": 0.0, "dgrad_conv": 0.0, "gram_fwd": 0.0, "gram_bwd": 0.0, "bwd_elementwise": 0.0, "other": 0.0}
    in_bwd = False
    for e in evs:
        n, t = e.name, e.device_time / 1e3
        if "percep_pack_net" in n:
            in_bwd = False
        if "percep_content_grad" in n or "percep_gram_diff" in n or "percep_mean_grad" in n:
            in_bwd = True
        if "conv_tc" in n:
            split["dgrad_conv" if in_bwd else "fwd_conv"] += t
        elif "percep_gram_grad" in n or "percep_gram_diff" in n:
            split["gram_bwd"] += t
        elif "percep_gram" in n:
            split["gram_fwd"] += t
        elif "percep_bwd" in n or "percep_content_grad" in n or "percep_grad_input" in n or "percep_mean_grad" in n:
            split["bwd_elementwise"] += t
        else:
            split["other"] += t
    split = {k: v / 3 for k, v in split.items()}
    flops, _ = percep_flops(mods, H, W, max(CONTENT + STYLE))
    dgrad_flops = flops * nimg  # the input-gradient convs mirror the stylized pass's convolutions
    return {"H": H, "W": W, "images": nimg, "ms_per_fwd_bwd": round(ms, 3),
            "kernel_ms": {k: round(v, 3) for k, v in split.items()},
            "dgrad_tflops": round(dgrad_flops / (split["dgrad_conv"] * 1e-3) / 1e12, 1) if split["dgrad_conv"] else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from fav_b200 import percep

    torch.cuda.set_device(0)
    mods = percep.vgg16_modules(0)
    crit = percep.PerceptualCriterion(mods, CONTENT, [1.0], STYLE, STYLE_W)
    yy, xx = np.mgrid[0:256, 0:256]
    style = np.stack([0.5 + 0.5 * np.sin(xx / 3.0 + c) * np.cos(yy / 5.0 - c) for c in range(3)]).astype(np.float32)
    crit.set_style_target(torch.from_numpy(style).cuda())
    res = {"card": card(),
           "train_256x256x4": measure(crit, mods, 256, 256, 4, args.steps, args.warmup),
           "frame_1280x720": measure(crit, mods, 720, 1280, 1, args.steps, args.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
