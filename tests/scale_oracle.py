"""fp64 restatement of image.scale(src, Wout, Hout, 'bicubic') and of run_image with -scale_factor.  TEST INFRASTRUCTURE ONLY.

image.scale belongs to the un-vendored `image` rock, so its arithmetic is not pinned here; this is the reading DESIGN.md §8
states (and csrc/scale.cu implements).  Two separable 1-D passes, x first: a line of n samples becomes m samples by
  m == n: a copy;
  else s = (float)(n-1)/(m-1), and for d = 0 .. m-2: t = d*s, i = min((int)t, n-2), f = t - i,
       p1 = src[i], p2 = src[i+1], p0 = i > 0 ? src[i-1] : 2*p1 - p2, p3 = i+2 < n ? src[i+2] : 2*p2 - p1,
       dst[d] = p1 + 0.5*f*((p2-p0) + f*((2*p0 - 5*p1 + 4*p2 - p3) + f*(3*(p1-p2) + p3 - p0)));
       dst[m-1] = src[n-1].
The sample positions s and t are computed in fp32, exactly as the reading does: an fp64 position differs from the fp32 one
by up to ~1e-4 px at 1280 samples, far above the kernel's bar.  The interpolation itself runs in fp64.

NetOracle extends oracle.net_oracle.NetOracle with the scale_factor of run_image (fast_artistic_video_core.lua:127-152).
"""
from __future__ import annotations

import numpy as np

from oracle import net_oracle


def positions(n: int, m: int):
    """(i, f) of output samples d = 0 .. m-2 of a line of n -> m samples: fp32 positions, i as int64, f as float32"""
    s = np.float32(n - 1) / np.float32(m - 1)
    t = np.arange(m - 1, dtype=np.float32) * s
    i = np.minimum(t.astype(np.int64), n - 2)
    return i, t - i.astype(np.float32)


def _scale_last_axis(a: np.ndarray, m: int) -> np.ndarray:
    n = a.shape[-1]
    if m == n:
        return a.copy()
    i, f32 = positions(n, m)
    f = f32.astype(np.float64)
    p1, p2 = a[..., i], a[..., i + 1]
    p0 = np.where(i > 0, a[..., np.maximum(i - 1, 0)], 2 * p1 - p2)
    p3 = np.where(i + 2 < n, a[..., np.minimum(i + 2, n - 1)], 2 * p2 - p1)
    out = np.empty(a.shape[:-1] + (m,), np.float64)
    out[..., :-1] = p1 + 0.5 * f * ((p2 - p0) + f * ((2 * p0 - 5 * p1 + 4 * p2 - p3) + f * (3 * (p1 - p2) + p3 - p0)))
    out[..., -1] = a[..., -1]
    return out


def image_scale_bicubic(src, Hout: int, Wout: int) -> np.ndarray:
    """src [..., Hin, Win] -> float64 [..., Hout, Wout]: the x pass, then the y pass.  A side of 1 is refused (ValueError): the
    reading has no step (n-1)/(m-1) for it."""
    a = np.asarray(src, dtype=np.float64)
    Hin, Win = a.shape[-2:]
    if min(Hin, Win, int(Hout), int(Wout)) < 2:
        raise ValueError(f"image_scale_bicubic: {Win}x{Hin} -> {Wout}x{Hout}: every side must be at least 2")
    a = _scale_last_axis(a, int(Wout))
    return np.swapaxes(_scale_last_axis(np.swapaxes(a, -1, -2), int(Hout)), -1, -2)


def _scale_last_axis_fp32(a: np.ndarray, m: int) -> np.ndarray:
    n = a.shape[-1]
    if m == n:
        return a.copy()
    f32 = np.float32
    i, f = positions(n, m)
    p1, p2 = a[..., i], a[..., i + 1]
    p0 = np.where(i > 0, a[..., np.maximum(i - 1, 0)], f32(2) * p1 - p2)
    p3 = np.where(i + 2 < n, a[..., np.minimum(i + 2, n - 1)], f32(2) * p2 - p1)
    a2 = ((f32(2) * p0 - f32(5) * p1) + f32(4) * p2) - p3
    a3 = (f32(3) * (p1 - p2) + p3) - p0
    out = np.empty(a.shape[:-1] + (m,), np.float32)
    out[..., :-1] = p1 + (f32(0.5) * f) * ((p2 - p0) + f * (a2 + f * a3))
    out[..., -1] = a[..., -1]
    return out


def image_scale_bicubic_fp32(src, Hout: int, Wout: int) -> np.ndarray:
    """The same reading as two fp32 passes (an fp32 intermediate [..., Hin, Wout]), every operation rounded to fp32 in the
    order written above: what the fused kernel must equal bit for bit."""
    a = np.ascontiguousarray(src, dtype=np.float32)
    a = _scale_last_axis_fp32(a, int(Wout))
    return np.swapaxes(_scale_last_axis_fp32(np.swapaxes(a, -1, -2), int(Hout)), -1, -2)


def scaled_size(H: int, W: int, scale_factor: float):
    h, w = H * scale_factor, W * scale_factor
    assert h == int(h) and w == int(w), (H, W, scale_factor)
    return int(h), int(w)


class NetOracle(net_oracle.NetOracle):
    def run_image(self, content01: np.ndarray, scale_factor: float = 1.0) -> np.ndarray:
        """fast_artistic_video_core.lua:121-158 with -scale_factor: scale the frame down (:127-129), run the image net at
        h x w (:146), deprocess (:149), scale back up (:150-152); the result is not clamped.  The scaled frame is rounded to
        fp32, as the image the net reads is."""
        if scale_factor == 1:
            return super().run_image(content01)
        assert self.in_dim == 3, "the video model cannot run a scaled frame (core.lua:133-138)"
        H, W = content01.shape[-2:]
        h, w = scaled_size(H, W, scale_factor)
        small = super().run_image(image_scale_bicubic(content01, h, w).astype(np.float32))
        return image_scale_bicubic(small, H, W)
