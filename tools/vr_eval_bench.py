"""-evaluate in the VR driver: (1) fav_vr_eval_gradient's kernel time and GB/s on a 2048x2048 face (torch.profiler, algorithmic
bytes 16 per pixel: three fp32 face planes and the fp32 mask); (2) ms per evaluated face, split into the VGG-16 loss network
and everything else (host clock around synchronised calls); (3) VR frames/s of tools/vr_bench.py's configuration (2048 px
faces, overlap 128, 3 VR frames, cube map + 2560x1440 equirect PNGs) with and without -evaluate, alternated over --repeats,
with a seeded VGG-16 .t7 and a 256 px style image.  Prints the card and its power limit with the numbers, one JSON line."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "fast-artistic-videos_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from fav_b200 import _lib, models_video, percep, synth, t7, vr  # noqa: E402

S, OV = 2048, 128
KERNELS = ("vr_eval_gradient_kernel", "vr_eval_finish_kernel")


def write_clip(d, nf):
    """tools/vr_bench.py's clip: six distinct faces repeated over nf VR frames, per-face flows and occlusion PGMs"""
    for f in range(1, nf + 1):
        for face in range(1, 7):
            src = f"{d}/src_{face}.ppm"
            if f == 1:
                synth.write_ppm(src, synth.make_frame(S, S, face))
            os.link(src, f"{d}/in_{f:03d}_{face}.ppm")
    for face in range(1, 7):
        synth.write_flo(f"{d}/src_bw_{face}.flo", synth.make_backward_flow(S, S, face + 1))
        rel = (np.random.default_rng(face).uniform(size=(S, S)) > 0.05).astype(np.uint8) * 255
        open(f"{d}/src_rel_{face}.pgm", "wb").write(b"P5\n%d %d\n255\n" % (S, S) + rel.tobytes())
        for f in range(2, nf + 1):
            os.link(f"{d}/src_bw_{face}.flo", f"{d}/bw_{f}_{f - 1}_{face}.flo")
            os.link(f"{d}/src_rel_{face}.pgm", f"{d}/rel_{f}_{f - 1}_{face}.pgm")


def kernel_bench(reps):
    face = torch.rand((3, S, S), device="cuda")
    mask = torch.rand((S, S), device="cuda")
    sums = torch.empty(6, dtype=torch.float64, device="cuda")
    call = lambda: _lib.check(_lib.lib.fav_vr_eval_gradient(_lib.dptr(face), _lib.dptr(mask), S, S, _lib.dptr(sums),
                                                            _lib.stream_ptr()))
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    us = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            for k in KERNELS:
                if k in ev.key:
                    us[k] = ev.device_time_total / ev.count
    assert set(us) == set(KERNELS), f"kernels missing from the profile: {us}"
    nbytes = 16 * S * S
    return {"gradient_kernel_us": round(us[KERNELS[0]], 2), "finish_kernel_us": round(us[KERNELS[1]], 2), "bytes": nbytes,
            "GB_per_s": round(nbytes / (us[KERNELS[0]] * 1e-6) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3, help="VR frames per timed run")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--reps", type=int, default=200, help="gradient-kernel launches in the profiled run")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vr_eval_bench needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    d = tempfile.mkdtemp(prefix="fav_vr_eval_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    try:
        write_clip(d, a.frames)
        t7.write_loss_network(f"{d}/vgg16.t7", percep.vgg16_modules(0))
        yy, xx = np.mgrid[0:256, 0:256]
        synth.write_ppm(f"{d}/style.ppm", np.stack([0.5 + 0.5 * np.sin(xx / 9.0 + c) * np.cos(yy / 13.0 - c)
                                                    for c in range(3)]).astype(np.float32))
        net = models_video.synthetic_model("mosaic", synth.PAPER_ARCH)
        argv = ["-input_pattern", f"{d}/in_%03d_%d.ppm", "-flow_pattern", f"{d}/bw_[%d]_{{%d}}_%d.flo",
                "-occlusions_pattern", f"{d}/rel_[%d]_{{%d}}_%d.pgm", "-output_prefix", f"{d}/out", "-overlap_pixel_w", str(OV),
                "-overlap_pixel_h", str(OV), "-out_equi", "-out_cubemap", "-out_equi_w", "2560", "-out_equi_h", "1440"]
        evaluate = ["-evaluate", "-evaluation_file", f"{d}/evaluation.txt", "-loss_network", f"{d}/vgg16.t7",
                    "-style_image", f"{d}/style.ppm"]
        configs = {"plain": argv, "evaluate": argv + evaluate}

        # (2) per-face split, from a 2-frame -evaluate run (the second frame has the temporal term)
        split = {"total": [], "vgg": []}
        orig_eval = vr.VRDriver.func_eval

        def timed_eval(self, opt, i, func_percept_loss, dtype):
            def percept(content, stylized):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = func_percept_loss(content, stylized)
                torch.cuda.synchronize()
                split["vgg"].append(time.perf_counter() - t0)
                return r

            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = orig_eval(self, opt, i, percept, dtype)
            torch.cuda.synchronize()
            split["total"].append(time.perf_counter() - t0)
            return r

        for cfg in configs.values():  # warm-up: plans, graphs, maps, the loss network
            vr.main(cfg + ["-num_frames", "1"], model_vid=net)
        vr.VRDriver.func_eval = timed_eval
        try:
            vr.main(configs["evaluate"] + ["-num_frames", "2"], model_vid=net)
        finally:
            vr.VRDriver.func_eval = orig_eval
        tot, vgg = np.array(split["total"]) * 1e3, np.array(split["vgg"]) * 1e3
        per_face = {"faces": len(tot), "ms_per_face_mean": round(float(tot.mean()), 3),
                    "vgg_ms_per_face_mean": round(float(vgg.mean()), 3),
                    "other_ms_per_face_mean": round(float((tot - vgg).mean()), 3),
                    "other_ms_per_face_min_max": [round(float((tot - vgg).min()), 3), round(float((tot - vgg).max()), 3)]}

        # (3) end to end, alternated
        fps = {k: [] for k in configs}
        for _ in range(a.repeats):
            for k, cfg in configs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                vr.main(cfg + ["-num_frames", str(a.frames)], model_vid=net)
                torch.cuda.synchronize()
                fps[k].append(a.frames / (time.perf_counter() - t0))
        e2e = {k: {"vr_frames_per_s_best": round(max(v), 3), "all": [round(x, 3) for x in v]} for k, v in fps.items()}

        # (1) the kernel alone, profiled in its own run
        kern = kernel_bench(a.reps)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    print(json.dumps({"card": card, "gradient_kernel_2048x2048": kern, "per_evaluated_face": per_face,
                      "vr_2048_ov128_e2e": e2e, "vr_frames": a.frames, "repeats": a.repeats}))


if __name__ == "__main__":
    main()
