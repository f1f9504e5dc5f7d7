"""Golden vectors of the REFERENCE's own CUDA warp kernel (run on an H100: `python tests/golden/make_warp_golden.py OUTDIR`).

oracle/_ref/libref_warp.so = stnbdhw/BilinearSamplerBDHW.cu:48-109 compiled for sm_90a (oracle/Makefile refwarp), built
where the reference sources are.  Writes
  OUTDIR/warp_ref.npz      outputs on the seeded inputs of WARP_CASES; committed as tests/golden/warp_ref.npz, pins
                           oracle/fav_oracle.c:orc_warp_bdhw on the CPU (tests/test_oracle.py) and the product on the GPU;
  OUTDIR/refwarp_cases.npz the reference kernel at the REF_SHAPES frame sizes (SHA-256 of every output plus a seeded
                           sample of its values), on batched / multi-channel / resized inputs, and the prior of the fused
                           temporal input composed from it; committed as tests/golden/refwarp_cases.npz
                           (tests/test_gpu_refwarp.py).
Inputs are regenerated from seeds at test time; only outputs are stored."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "fast-artistic-videos_b200"))

from fav_b200 import synth  # noqa: E402

WARP_CASES = [  # (name, C, Hin, Win, Hout, Wout, flow kind)
    ("real_64x96", 3, 64, 96, 64, 96, "real"), ("stress_64x96", 3, 64, 96, 64, 96, "stress"),
    ("real_97x75", 3, 97, 75, 97, 75, "real"), ("stress_33x129", 1, 33, 129, 33, 129, "stress"),
    ("resize_40x56_to_52x44", 5, 40, 56, 52, 44, "rand"), ("sentinel_32x48", 1, 32, 48, 32, 48, "sentinel")]


def warp_inputs(case):
    name, C, Hin, Win, Ho, Wo, kind = case
    rng = np.random.default_rng(sum(map(ord, name)))
    if C == 3:
        img = synth.make_frame(Hin, Win, 1) * 1.2 - 0.1
    else:
        img = rng.uniform(-0.2, 1.2, size=(C, Hin, Win)).astype(np.float32)
    if kind == "real":
        flow = synth.checker_to_lua(synth.make_backward_flow(Ho, Wo, 2))
    elif kind == "stress":
        flow = synth.stress_flow(Ho, Wo)
    elif kind == "sentinel":  # vr_helper.lua:10 maps: 99999 outside the strip, a real offset inside
        flow = np.full((2, Ho, Wo), 99999.0, np.float32)
        flow[:, :, Wo // 3: Wo // 2] = rng.uniform(-5, 5, size=(2, Ho, Wo // 2 - Wo // 3)).astype(np.float32)
    else:
        flow = rng.uniform(-9, 9, size=(2, Ho, Wo)).astype(np.float32)
    return np.ascontiguousarray(img, np.float32), np.ascontiguousarray(flow, np.float32)


# the five BASELINE.json config shapes (256^2 tiny, 720p, 1080p, 2048^2 VR face, 4K) + ragged small ones
REF_SHAPES = [(256, 256), (720, 1280), (1080, 1920), (2048, 2048), (2160, 3840), (97, 75), (33, 129)]
N_SAMPLE = 1024


def shape_inputs(H, W):
    img = synth.make_frame(H, W, 1) * 1.2 - 0.1
    flows = {"real": synth.checker_to_lua(synth.make_backward_flow(H, W, 2)), "stress": synth.stress_flow(H, W)}
    return np.ascontiguousarray(img, np.float32), flows


def batch_inputs():
    rng = np.random.default_rng(0)
    img = rng.uniform(size=(2, 5, 20, 28)).astype(np.float32)
    grid = rng.uniform(-6, 6, size=(2, 2, 13, 36)).astype(np.float32)
    return img, grid


def prior_inputs():
    from oracle import net_oracle

    H, W = 360, 640
    return (synth.make_frame(H, W, 2), synth.make_frame(H, W, 1) * 1.2 - 0.1,
            synth.checker_to_lua(synth.make_backward_flow(H, W, 2)), net_oracle.make_cert(H, W, 2))


def compose_prior(warped, cert):
    """preprocess(warp) * cert in the reference's op order (core.lua:166-167), on torch tensors."""
    import torch

    mean = torch.tensor([103.939, 116.779, 123.68], device=warped.device).view(3, 1, 1)
    pre = warped[[2, 1, 0]] * 255.0 - mean           # preprocess.lua:57-62: index, mul(255), add(-1, mean)
    return torch.zeros_like(pre) + pre * cert        # core.lua:167 fill(vgg-mean = 0) + cmul


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def sample_index(n):
    return np.random.default_rng(n).choice(n, size=min(N_SAMPLE, n), replace=False)


def main(outdir):
    import torch

    from oracle import refwarp

    def T(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    out = {}
    for case in WARP_CASES:
        img, flow = warp_inputs(case)
        out[case[0]] = refwarp.warp(T(img)[None], T(flow)[None])[0].cpu().numpy()
    os.makedirs(outdir, exist_ok=True)
    np.savez_compressed(os.path.join(outdir, "warp_ref.npz"), **out)
    cases = {}
    for H, W in REF_SHAPES:
        img, flows = shape_inputs(H, W)
        for name, flow in flows.items():
            o = refwarp.warp(T(img)[None], T(flow)[None])[0].cpu().numpy()
            key = f"{H}x{W}_{name}"
            cases[key + "_sha"] = np.array(digest(o))
            cases[key + "_sample"] = o.reshape(-1)[sample_index(o.size)]
    img, grid = batch_inputs()
    cases["batch"] = refwarp.warp(T(img), T(grid)).cpu().numpy()
    cases["sentinel"] = refwarp.warp(T(img[:1]), torch.full((1, 2, 20, 28), 99999.0, device="cuda")).cpu().numpy()
    c, p, flow, cert = prior_inputs()
    cases["prior_360x640_sha"] = np.array(digest(compose_prior(refwarp.warp(T(p)[None], T(flow)[None])[0], T(cert)).cpu().numpy()))
    np.savez_compressed(os.path.join(outdir, "refwarp_cases.npz"), **cases)
    print("wrote", outdir, "warp_ref.npz", "refwarp_cases.npz", len(cases), "entries")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else ".")
