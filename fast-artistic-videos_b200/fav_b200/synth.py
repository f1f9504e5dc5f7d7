"""Seeded synthetic inputs and weights (SURVEY.md §8(d)).

The reference ships neither test data nor weights (`models/download_models.sh` needs a network),
so every parity/bench run uses the generators below.  Pure numpy, deterministic, little-endian
fp32.  This module is DATA ONLY - it contains none of the hot-path arithmetic.

Weights follow Torch7's own module initialisers, which is what a freshly built
`models_video.build_model` (fast_artistic_video/models_video.lua:55-140) holds:
  nn.SpatialConvolution / SpatialFullConvolution reset(): U(-s, s), s = 1/sqrt(kW*kH*nInputPlane)
  nn.InstanceNormalization: weight ~ U[0,1), bias = 0   (InstanceNormalization.lua:26-27)
  nn.SpatialBatchNormalization (norm='batch'): the same, plus running_mean = 0, running_var = 1, eps = 1e-5
One seed per style name ("candy", "mosaic", "scream", ...).
"""
from __future__ import annotations

import zlib

import numpy as np

DEFAULT_ARCH = "c9s1-32,d64,d128,R128,R128,R128,R128,R128,u64,u32,c9s1-3"  # train_video.lua:21
PAPER_ARCH = "c9s1-32,d64,d128,R128,R128,R128,R128,R128,U2,c3s1-64,U2,c9s1-3"  # README.md:256


def style_seed(style: str) -> int:
    return zlib.crc32(style.encode()) & 0x7FFFFFFF


def parse_arch(arch: str, in_dim: int = 7):
    """Token list of models_video.build_model (models_video.lua:59-133) -> list of layer specs.

    Each spec: dict(kind=..., cin, cout, k, stride, pad, in_norm, relu).  'R' expands to one spec
    of kind 'res' (two 3x3 pad-0 convs + IN, ShaveImage(2) skip: build_res_block :41-53 with
    padding_type 'reflect-start').
    """
    toks = arch.split(",")
    specs = []
    prev = in_dim
    for i, v in enumerate(toks):
        c0 = v[0]
        needs_bn = needs_relu = True
        if c0 == "c":  # :65-80
            f = int(v[1]); s = int(v[3]); nxt = int(v[5:])
            spec = dict(kind="conv", cin=prev, cout=nxt, k=f, stride=s, pad=(f - 1) // 2)
        elif c0 == "f":  # :81-89
            f = int(v[1]); s = int(v[3]); nxt = int(v[5:])
            spec = dict(kind="fullconv", cin=prev, cout=nxt, k=f, stride=s, pad=(f - 1) // 2, adj=s - 1)
        elif c0 == "d":  # :90-93
            nxt = int(v[1:])
            spec = dict(kind="conv", cin=prev, cout=nxt, k=3, stride=2, pad=1)
        elif c0 == "U":  # :94-98
            nxt = prev
            spec = dict(kind="up", cin=prev, cout=nxt, scale=int(v[1:]))
        elif c0 == "u":  # :99-102
            nxt = int(v[1:])
            spec = dict(kind="fullconv", cin=prev, cout=nxt, k=3, stride=2, pad=1, adj=1)
        elif c0 == "R":  # :109-114
            nxt = int(v[1:])
            spec = dict(kind="res", cin=prev, cout=nxt, k=3, stride=1, pad=0, skip=True)
            needs_bn = needs_relu = False
        elif c0 == "C":  # :103-108: the conv block of a residual block without the skip, ReLU after it
            nxt = int(v[1:])
            spec = dict(kind="res", cin=prev, cout=nxt, k=3, stride=1, pad=0, skip=False)
            needs_bn = False
        else:
            raise ValueError(f"unsupported arch token {v!r}")
        if i == len(toks) - 1:  # :117-120
            needs_bn = needs_relu = False
        spec["in_norm"] = needs_bn
        spec["relu"] = needs_relu
        specs.append(spec)
        prev = nxt
    return specs


def reflect_start_pad(specs, padding_type: str = "reflect-start") -> int:
    """Padding that train_video.lua:319-324 lazily inserts as layer 1 (reflect-start): half of what the unpadded blocks shave."""
    if padding_type != "reflect-start":
        return 0
    # track (scale numerator) shrink in input pixels: each res block loses 4 px at its resolution
    scale = 1.0
    shrink = 0.0
    for s in specs:
        if s["kind"] == "conv" and s["stride"] == 2:
            scale *= 2
        elif s["kind"] == "fullconv" and s["stride"] == 2:
            scale /= 2
        elif s["kind"] == "up":
            scale /= s["scale"]
        elif s["kind"] == "res":
            shrink += 4 * scale
    assert shrink == int(shrink) and int(shrink) % 2 == 0
    return int(shrink) // 2


def make_weights(arch: str = DEFAULT_ARCH, style: str = "candy", in_dim: int = 7, norm: str = "instance"):
    """Dict name -> fp32 array.  conv: (cout,cin,k,k); fullconv: (cin,cout,k,k) (Torch layout).  norm='batch' adds each norm's
    running statistics and eps; every other array (and the random stream) is the one norm='instance' gives."""
    assert norm in ("instance", "batch")
    rng = np.random.default_rng(style_seed(style))
    specs = parse_arch(arch, in_dim)
    w = {}

    def conv_w(name, cin, cout, k, transposed=False):
        s = 1.0 / np.sqrt(k * k * cin)
        shape = (cin, cout, k, k) if transposed else (cout, cin, k, k)
        w[name + ".weight"] = rng.uniform(-s, s, size=shape).astype(np.float32)
        w[name + ".bias"] = rng.uniform(-s, s, size=(cout,)).astype(np.float32)

    def in_w(name, c):
        w[name + ".weight"] = rng.uniform(0.0, 1.0, size=(c,)).astype(np.float32)
        w[name + ".bias"] = np.zeros((c,), np.float32)
        if norm == "batch":
            w[name + ".running_mean"] = np.zeros((c,), np.float32)
            w[name + ".running_var"] = np.ones((c,), np.float32)
            w[name + ".eps"] = np.full((1,), 1e-5, np.float32)

    for i, s in enumerate(specs):
        n = f"l{i}"
        if s["kind"] == "conv":
            conv_w(n, s["cin"], s["cout"], s["k"])
        elif s["kind"] == "fullconv":
            conv_w(n, s["cin"], s["cout"], s["k"], transposed=True)
        elif s["kind"] == "res":
            conv_w(n + ".c1", s["cin"], s["cout"], 3); in_w(n + ".n1", s["cout"])
            conv_w(n + ".c2", s["cout"], s["cout"], 3); in_w(n + ".n2", s["cout"])
        if s["in_norm"]:
            in_w(n + ".n", s["cout"])
    return w


# ---------------------------------------------------------------------------------------------
# clips: frames, backward/forward flow (SURVEY.md §8(d))
# ---------------------------------------------------------------------------------------------
def _coords(H, W):
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return y, x


def make_frame(H: int, W: int, idx: int) -> np.ndarray:
    """3xHxW RGB in [0,1]: smooth sinusoid base translated by the clip motion + 5% noise."""
    rng = np.random.default_rng(1000 + idx)
    y, x = _coords(H, W)
    tx, ty = 3.25 * idx, -1.5 * idx
    img = np.empty((3, H, W), np.float64)
    for c, (fx, fy, ph) in enumerate([(3.0, 2.0, 0.3), (5.0, 1.0, 1.1), (2.0, 4.0, 2.3)]):
        img[c] = 0.5 + 0.45 * np.sin(2 * np.pi * (fx * (x - tx) / W + fy * (y - ty) / H) + ph)
    img += 0.05 * rng.uniform(-1, 1, size=img.shape)
    return np.clip(img, 0.0, 1.0).astype(np.float32)


def make_backward_flow(H: int, W: int, idx: int) -> np.ndarray:
    """Flow i -> i-1 in CHECKER layout (plane 0 = u / dx, plane 1 = v / dy), fp32 [2,H,W]."""
    rng = np.random.default_rng(2000 + idx)
    y, x = _coords(H, W)
    ph = rng.uniform(0, 2 * np.pi, size=2)
    u = -3.25 + 4.0 * np.sin(2 * np.pi * y / H + ph[0]) * np.cos(2 * np.pi * x / W)
    v = 1.5 + 4.0 * np.cos(2 * np.pi * x / W + ph[1]) * np.sin(2 * np.pi * y / H)
    bs = max(8, int(round(64 * W / 1280)))  # independently moving block -> real occlusions
    y0 = int(rng.integers(H // 8, max(H // 8 + 1, H - bs - H // 8)))
    x0 = int(rng.integers(W // 8, max(W // 8 + 1, W - bs - W // 8)))
    u[y0:y0 + bs, x0:x0 + bs] += 9.0
    v[y0:y0 + bs, x0:x0 + bs] += -6.0
    return np.stack([u, v]).astype(np.float32)


def make_forward_flow(H: int, W: int, idx: int) -> np.ndarray:
    """Flow i-1 -> i: negated backward flow resampled at the target + N(0,0.05) noise (checker layout)."""
    rng = np.random.default_rng(3000 + idx)
    bw = make_backward_flow(H, W, idx).astype(np.float64)
    y, x = _coords(H, W)
    # crude inverse: f_fw(p) ~= -f_bw(p - f_bw(p)) (nearest sample)
    sx = np.clip(np.rint(x - bw[0]), 0, W - 1).astype(np.int64)
    sy = np.clip(np.rint(y - bw[1]), 0, H - 1).astype(np.int64)
    fw = -bw[:, sy, sx]
    fw += rng.normal(0.0, 0.05, size=fw.shape)
    return np.ascontiguousarray(fw, dtype=np.float32)


def stress_flow(H: int, W: int, seed: int = 7, amp: float = 64.0) -> np.ndarray:
    """i.i.d. U(-amp, amp) px flow in LUA layout (ch0 = dy, ch1 = dx): worst-case gather locality."""
    rng = np.random.default_rng(seed)
    return rng.uniform(-amp, amp, size=(2, H, W)).astype(np.float32)


def checker_to_lua(flow_uv: np.ndarray) -> np.ndarray:
    """(u,v) planes -> flowFileLoader layout [dy, dx] (flowFileLoader.lua:31-32)."""
    return np.ascontiguousarray(flow_uv[::-1])


def write_flo(path: str, flow_uv: np.ndarray) -> None:
    """Middlebury .flo: tag 202021.25, int32 W, int32 H, interleaved (u,v) fp32 (flowFileLoader.lua:8-15)."""
    _, H, W = flow_uv.shape
    with open(path, "wb") as f:
        np.array([202021.25], np.float32).tofile(f)
        np.array([W, H], np.int32).tofile(f)
        np.ascontiguousarray(np.transpose(flow_uv, (1, 2, 0)), dtype=np.float32).tofile(f)


def write_ppm(path: str, rgb01: np.ndarray) -> None:
    """3xHxW [0,1] -> binary P6 (what ffmpeg extracts and image.load / readFromPPM consume)."""
    _, H, W = rgb01.shape
    u8 = np.clip(np.rint(rgb01 * 255.0), 0, 255).astype(np.uint8)
    with open(path, "wb") as f:
        f.write(b"P6\n%d %d\n255\n" % (W, H))
        np.ascontiguousarray(np.transpose(u8, (1, 2, 0))).tofile(f)


def read_pgm(path: str) -> np.ndarray:
    with open(path, "rb") as f:
        data = f.read()
    # "P5\n%d %d\n255\n" (CMatrix.h:1064)
    parts = data.split(b"\n", 3)
    assert parts[0] == b"P5", parts[0]
    W, H = (int(t) for t in parts[1].split())
    assert parts[2] == b"255"
    return np.frombuffer(parts[3], np.uint8, count=W * H).reshape(H, W).copy()
