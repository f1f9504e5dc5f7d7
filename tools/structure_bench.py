"""The checker's 4-argument mode on the GPU: per-kernel time of fav_compute_corners (the exact average's kernels separately) at
720p, 1080p, 2048^2 and 4K, frames/s of run_next_image_flows in 3- versus 4-argument mode (alternated) at 720p and 1080p, and
end-to-end frames/s of the native file pipeline from files at 720p (PPM + .flo + certainty PGM versus PPM + both .flo, alternated;
the clip is written to a temporary directory).  Prints the card and its power limit with the numbers, one JSON line.  --lib PATH also times fav_compute_corners of another
build of libfav_b200.so in the same process (CUDA events, whole call)."""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "fast-artistic-videos_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from fav_b200 import _lib, models_video, synth  # noqa: E402

SIZES = {"720p": (720, 1280), "1080p": (1080, 1920), "2048sq": (2048, 2048), "4k": (2160, 3840)}
AVG_KERNELS = ("avg_sum_kernel", "avg_hyp_kernel", "avg_walk_kernel")


def frame255(H, W, idx=2):
    img = np.clip(np.rint(synth.make_frame(H, W, idx) * 255.0), 0, 255).astype(np.float32)
    img[:, :, : W // 3] = 128.0  # a flat third, as in the tests
    return torch.from_numpy(img).cuda()


def corners_call(lib, img, corners, avg, ws):
    Z, H, W = img.shape
    rc = lib.fav_compute_corners(C.c_void_p(img.data_ptr()), Z, W, H, C.c_float(3.0), C.c_void_p(corners.data_ptr()),
                                 C.c_void_p(avg.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_void_p(0))
    assert rc == 0, rc


def time_events(fn, reps):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def corners_bench(other, reps):
    out = {}
    lib = _lib.lib
    for name, (H, W) in SIZES.items():
        img = frame255(H, W)
        corners = torch.empty((H, W), device="cuda")
        avg = torch.empty((1,), device="cuda")
        ws = torch.empty(int(lib.fav_compute_corners_workspace(3, W, H)), dtype=torch.uint8, device="cuda")
        r = {"call_ms": time_events(lambda: corners_call(lib, img, corners, avg, ws), reps)}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                corners_call(lib, img, corners, avg, ws)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "kernel" in ev.key:
                per[ev.key.split("(")[0].split("::")[-1]] = ev.device_time_total / 1e3 / reps
        r["kernels_ms"] = {k: round(v, 4) for k, v in sorted(per.items())}
        r["avg_kernels_ms"] = round(sum(v for k, v in per.items() if k in AVG_KERNELS), 4)
        r["other_kernels_ms"] = round(sum(v for k, v in per.items() if k not in AVG_KERNELS), 4)
        if other is not None:
            ows = torch.empty(int(other.fav_compute_corners_workspace(3, W, H)), dtype=torch.uint8, device="cuda")
            oavg = torch.empty((1,), device="cuda")
            r["other_lib_call_ms"] = time_events(lambda: corners_call(other, img, corners, oavg, ows), max(3, reps // 4))
            r["same_average_bits"] = bool(torch.equal(avg.view(torch.int32), oavg.view(torch.int32)))
        out[name] = r
    return out


def frames_bench(frames, rounds):
    net = models_video.synthetic_model("candy")
    out = {}
    for name in ("720p", "1080p"):
        H, W = SIZES[name]
        x = torch.from_numpy(synth.make_frame(H, W, 2)).cuda()
        p = torch.from_numpy(synth.make_frame(H, W, 1)).cuda()
        f = torch.from_numpy(synth.checker_to_lua(synth.make_backward_flow(H, W, 2))).cuda()
        fw = torch.from_numpy(synth.make_forward_flow(H, W, 2)).cuda()
        modes = {"3arg": lambda: net.run_next_image_flows(x, p, f, fw, None, 7),
                 "4arg": lambda: net.run_next_image_flows_structure(x, p, f, fw, 7)}
        res = {k: [] for k in modes}
        for _ in range(rounds):
            for k, fn in modes.items():
                res[k].append(1e3 / time_events(fn, frames))
        out[name] = {k: {"fps_best": round(max(v), 1), "fps_all": [round(a, 1) for a in v]} for k, v in res.items()}
    return out


def files_bench(frames, rounds):
    """video.run_native on a 720p clip: certainty PGMs (fav_video_pipeline_run) vs forward flows (fav_video_pipeline_run_flows)."""
    from fav_b200 import consistencyChecker, video

    H, W = SIZES["720p"]
    d = tempfile.mkdtemp(prefix="fav_structure_bench_")
    try:
        pool = 4  # distinct frames / flows, linked under the per-frame names
        for k in range(pool):
            synth.write_ppm(f"{d}/src_frame_{k}.ppm", synth.make_frame(H, W, k + 1))
            bw, fw = synth.make_backward_flow(H, W, k + 2), synth.make_forward_flow(H, W, k + 2)
            synth.write_flo(f"{d}/src_bw_{k}.flo", bw)
            synth.write_flo(f"{d}/src_fw_{k}.flo", fw)
            img = torch.from_numpy(consistencyChecker.read_ppm_planes(f"{d}/src_frame_{k}.ppm")).cuda()
            rel = consistencyChecker.check(torch.from_numpy(bw).cuda(), torch.from_numpy(fw).cuda(), img).cpu().numpy()
            open(f"{d}/src_rel_{k}.pgm", "wb").write(b"P5\n%d %d\n255\n" % (W, H) + rel.tobytes())
        for i in range(1, frames + 1):
            os.link(f"{d}/src_frame_{i % pool}.ppm", f"{d}/frame_{i:04d}.ppm")
            if i > 1:
                os.link(f"{d}/src_bw_{i % pool}.flo", f"{d}/backward_{i}_{i - 1}.flo")
                os.link(f"{d}/src_fw_{i % pool}.flo", f"{d}/forward_{i - 1}_{i}.flo")
                os.link(f"{d}/src_rel_{i % pool}.pgm", f"{d}/reliable_{i}_{i - 1}.pgm")
        net = models_video.synthetic_model("candy")
        common = ["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo", "-num_frames",
                  str(frames), "-output_prefix", f"{d}/out"]
        opts = {"pgm": video.build_parser().parse_args(common + ["-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm"]),
                "flows": video.build_parser().parse_args(common + ["-flow_pattern_forward", f"{d}/forward_{{%d}}_[%d].flo"])}
        res = {k: [] for k in opts}
        for o in opts.values():
            video.run_native(o, model_vid=net)  # warm: page cache, plans, graphs
        for _ in range(rounds):
            for k, o in opts.items():
                r = video.run_native(o, model_vid=net)
                res[k].append(r["frames"] / r["seconds"])
        return {k: {"fps_best": round(max(v), 1), "fps_all": [round(a, 1) for a in v]} for k, v in res.items()} | {
            "frames": frames, "cpus": os.cpu_count()}
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="another libfav_b200.so whose fav_compute_corners is timed alongside")
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--clip-frames", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "structure_bench needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    other = None
    if a.lib:
        other = C.CDLL(os.path.abspath(a.lib))
        other.fav_compute_corners_workspace.restype = C.c_size_t
    res = {"card": card, "corners": corners_bench(other, a.reps), "run_next_image_flows": frames_bench(a.frames, a.rounds),
           "files_720p": files_bench(a.clip_frames, a.rounds)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
