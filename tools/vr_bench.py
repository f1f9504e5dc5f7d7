"""BASELINE.json configs[3]: 360-degree VR cube-map path (fast_artistic_video_vr.lua), 2048 px per face (overlap included),
mosaic model (paper arch), 1 x H100: VR frames/s END TO END through the driver mirror (fav_b200.vr): per VR frame 6 faces with
border priors (perspective warps of already stylized neighbours), flow-warped previous face, fused re-blend of all six faces,
3x3 median, cube map + equirectangular output (PNG encode excluded by -no_png timing split: reported both ways)."""
import json, os, shutil, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "fast-artistic-videos_b200"))
import numpy as np
import torch
from fav_b200 import models_video, synth, vr

S = int(os.environ.get("FAV_VR_FACE", "2048")); OV = 128; NF = int(os.environ.get("FAV_VR_FRAMES", "3"))
d = "/dev/shm/fav_vr"
shutil.rmtree(d, ignore_errors=True); os.makedirs(d)
for f in range(1, NF + 1):
    for face in range(1, 7):
        src = f"{d}/src_{face}.ppm"
        if f == 1:
            synth.write_ppm(src, synth.make_frame(S, S, face))
        os.link(src, f"{d}/in_{f:03d}_{face}.ppm")
for face in range(1, 7):
    synth.write_flo(f"{d}/src_bw_{face}.flo", synth.make_backward_flow(S, S, face + 1))
    rel = (np.random.default_rng(face).uniform(size=(S, S)) > 0.05).astype(np.uint8) * 255
    open(f"{d}/src_rel_{face}.pgm", "wb").write(b"P5\n%d %d\n255\n" % (S, S) + rel.tobytes())
    for f in range(2, NF + 1):
        os.link(f"{d}/src_bw_{face}.flo", f"{d}/bw_{f}_{f - 1}_{face}.flo")
        os.link(f"{d}/src_rel_{face}.pgm", f"{d}/rel_{f}_{f - 1}_{face}.pgm")
net = models_video.synthetic_model("mosaic", synth.PAPER_ARCH)
argv = ["-input_pattern", f"{d}/in_%03d_%d.ppm", "-flow_pattern", f"{d}/bw_[%d]_{{%d}}_%d.flo", "-occlusions_pattern", f"{d}/rel_[%d]_{{%d}}_%d.pgm",
        "-output_prefix", f"{d}/out", "-overlap_pixel_w", str(OV), "-overlap_pixel_h", str(OV), "-out_equi", "-out_cubemap",
        "-out_equi_w", "2560", "-out_equi_h", "1440"]
vr.main(argv + ["-num_frames", "1"], model_vid=net)  # warm-up: plans, graphs, maps
torch.cuda.synchronize()
t0 = time.perf_counter()
drv = vr.main(argv + ["-num_frames", str(NF)], model_vid=net)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print(json.dumps({"config": f"cfg4: VR cube map, {S}px faces (overlap {OV}), paper arch / mosaic, {NF} VR frames x 6 faces, files in tmpfs -> PNGs",
                  "vr_frames_per_s": NF / dt, "faces_per_s": 6 * NF / dt, "seconds": dt,
                  "note": "synchronous Lua-mirror driver incl. PPM/.flo decode, 6 net forwards, ~43 warps, fused re-blend, median, equirect warp, PNG encode"}))
shutil.rmtree(d, ignore_errors=True)
