"""-scale_factor: ms per 1280x720 run_image of a 3-channel image model at scale factors 1, 0.5 and 2 (CUDA events, the three
alternated, --steps calls x --repeats), and, in a separate torch.profiler run, the bicubic resampler's kernel time and
achieved GB/s (algorithmic bytes 4*C*(Hin*Win + Hout*Wout)) for 720p -> 360p and 360p -> 720p.  Prints the card and its power
limit with the numbers, one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "fast-artistic-videos_b200"))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from fav_b200 import _lib, models_video, synth  # noqa: E402

H, W = 720, 1280
FACTORS = (1.0, 0.5, 2.0)
RESAMPLES = {"720p_to_360p": ((720, 1280), (360, 640)), "360p_to_720p": ((360, 640), (720, 1280))}
KERNEL = "scale_bicubic_kernel"


def time_events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def run_image_bench(steps, repeats, warmup):
    net = models_video.synthetic_model("candy", synth.DEFAULT_ARCH, in_dim=3)
    x = torch.from_numpy(synth.make_frame(H, W, 1)).cuda()
    res = {sf: [] for sf in FACTORS}
    for _ in range(repeats):
        for sf in FACTORS:
            res[sf].append(time_events(lambda: net.run_image(x, scale_factor=sf), steps, warmup))
    return {f"sf_{sf:g}": {"ms_best": round(min(v), 4), "ms_all": [round(a, 4) for a in v]} for sf, v in res.items()}


def resample_bench(reps):
    out = {}
    for name, ((hi, wi), (ho, wo)) in RESAMPLES.items():
        src = torch.rand((3, hi, wi), device="cuda")
        dst = torch.empty((3, ho, wo), device="cuda")
        call = lambda: _lib.check(_lib.lib.fav_image_scale_bicubic(_lib.dptr(src), _lib.dptr(dst), 3, hi, wi, ho, wo,
                                                                      _lib.stream_ptr()))
        call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        us = [ev.device_time_total / ev.count for ev in prof.key_averages()
              if ev.device_type == torch.autograd.DeviceType.CUDA and KERNEL in ev.key]
        assert len(us) == 1, f"{KERNEL} not found in the profile"
        nbytes = 4 * 3 * (hi * wi + ho * wo)
        out[name] = {"kernel_us": round(us[0], 3), "bytes": nbytes, "GB_per_s": round(nbytes / (us[0] * 1e-6) / 1e9, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200, help="resampler launches in the profiled run")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "scale_bench needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"card": card, "run_image_1280x720_ms": run_image_bench(a.steps, a.repeats, a.warmup),
           "resampler": resample_bench(a.reps)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
