"""PyTorch-CPU restatement of the stylization net and the frame loop.  TEST INFRASTRUCTURE ONLY.

Follows (reference file:line):
  models_video.build_model            fast_artistic_video/models_video.lua:55-140
  build_res_block / build_conv_block  models_video.lua:10-53   (reflect-start: pad-0 convs + ShaveImage(2))
  nn.InstanceNormalization            InstanceNormalization.lua:33-53 (batch-stat BN over 1x(N*C)xHxW,
                                      eps 1e-5, biased variance, always training mode :49)
  nn.ShaveImage                       ShaveImage.lua:9-16
  lazily inserted ReflectionPadding   train_video.lua:316-325
  Tanh, MulConstant(150), TV(identity) models_video.lua:135-137, TotalVariation.lua:12-15
  run_image / run_next_image          fast_artistic_video_core.lua:121-180

The layer arithmetic itself lives in un-vendored, unpinned Torch7 rocks (nn / cunn / cudnn):
PARITY UNPINNED at that boundary; the well-known Torch7 semantics are restated with
F.conv2d / F.conv_transpose2d(stride 2, padding 1, output_padding 1; same in x out x k x k weight
layout as nn.SpatialFullConvolution) / F.instance_norm(eps=1e-5) / F.pad(reflect) / nearest upsampling.
fp64 = ground truth, fp32 = "reference precision" comparator.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fast-artistic-videos_b200")
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)
from fav_b200 import synth  # noqa: E402  (data generators only)

from . import pyoracle  # noqa: E402

VGG_MEAN = (103.939, 116.779, 123.68)  # preprocess.lua:48


def _inorm(x, w, name):
    # InstanceNormalization.lua:33-53
    return F.instance_norm(x, weight=w[name + ".weight"], bias=w[name + ".bias"], eps=1e-5)


class NetOracle:
    def __init__(self, arch=synth.DEFAULT_ARCH, style="candy", dtype=torch.float64, weights=None,
                 tanh_constant=150.0, operand_round=None, in_dim=7, padding_type="reflect-start"):
        assert padding_type in ("reflect-start", "zero")  # models_video.lua:13-19,46-50
        self.specs = synth.parse_arch(arch, in_dim)
        self.pad = synth.reflect_start_pad(self.specs, padding_type)
        self.block_pad = 1 if padding_type == "zero" else 0
        self.in_dim = in_dim
        wnp = weights if weights is not None else synth.make_weights(arch, style, in_dim)
        self.w = {k: torch.from_numpy(v).to(dtype) for k, v in wnp.items()}
        self.dtype = dtype
        self.tanh_constant = tanh_constant
        # operand_round: optional callable emulating reduced-precision MMA operands (experiments only)
        self.operand_round = operand_round

    def _conv(self, x, name, stride, pad):
        wt, b = self.w[name + ".weight"], self.w[name + ".bias"]
        if self.operand_round is not None:
            return self.operand_round(x, wt, b, dict(stride=stride, padding=pad), False)
        return F.conv2d(x, wt, b, stride=stride, padding=pad)

    def _fullconv(self, x, name, s):
        wt, b = self.w[name + ".weight"], self.w[name + ".bias"]
        kw = dict(stride=s["stride"], padding=s["pad"], output_padding=s["adj"])
        if self.operand_round is not None:
            return self.operand_round(x, wt, b, kw, True)
        return F.conv_transpose2d(x, wt, b, **kw)

    def to(self, device) -> "NetOracle":
        """Moves the weights to `device` (e.g. "cuda": cuDNN in fp64 for frames a CPU forward cannot reach); layer and forward
        then take inputs on that device."""
        self.w = {k: v.to(device) for k, v in self.w.items()}
        return self

    def layer(self, i: int, x: torch.Tensor, norm_hook=None) -> torch.Tensor:
        """Arch token i's step on x, the output of step i - 1 (for i = 0 the 1xCxHxW net input, which the reflect-start
        padding then pads): conv / transposed conv / nearest upsample / residual block, then InstanceNorm and ReLU.
        norm_hook(name, t): optional, called with the input t of each InstanceNorm the step runs."""
        s, n = self.specs[i], f"l{i}"
        x = x.to(self.dtype)

        def inorm(t, name):
            if norm_hook is not None:
                norm_hook(name, t)
            return _inorm(t, self.w, name)

        if i == 0 and self.pad:
            x = F.pad(x, (self.pad,) * 4, mode="reflect")  # train_video.lua:322
        if s["kind"] == "conv":
            x = self._conv(x, n, s["stride"], s["pad"])
        elif s["kind"] == "fullconv":
            x = self._fullconv(x, n, s)
        elif s["kind"] == "up":
            x = F.interpolate(x, scale_factor=s["scale"], mode="nearest")
        elif s["kind"] == "res":  # build_conv_block :10-39 (+ ConcatTable / CAddTable :41-53 for RX)
            bp = self.block_pad
            y = self._conv(x, n + ".c1", 1, bp)
            y = torch.relu(inorm(y, n + ".n1"))
            y = self._conv(y, n + ".c2", 1, bp)
            y = inorm(y, n + ".n2")
            if not s.get("skip", True):
                x = y                                    # CX
            elif bp:
                x = y + x                                # Identity skip ('zero')
            else:
                x = y + x[:, :, 2:-2, 2:-2]              # ShaveImage(2) + CAddTable
        if s["in_norm"]:
            x = inorm(x, n + ".n")
        if s["relu"]:
            x = torch.relu(x)
        return x

    def forward(self, x7: torch.Tensor, taps=None) -> torch.Tensor:
        """x7: 1x7xHxW -> 1x3xHxW (net space, before deprocess).  taps: optional dict to record activations."""
        x = x7
        for i in range(len(self.specs)):
            x = self.layer(i, x)
            if taps is not None:
                taps[f"l{i}"] = x
        return torch.tanh(x) * self.tanh_constant  # models_video.lua:135-136

    # --- frame-level restatements -----------------------------------------------------------
    def deprocess(self, y):  # preprocess.lua:66-71
        mean = torch.tensor(VGG_MEAN, dtype=self.dtype, device=y.device).view(1, 3, 1, 1)
        return ((y + mean) / 255.0)[:, [2, 1, 0]]

    def run_image(self, content01: np.ndarray) -> np.ndarray:
        """fast_artistic_video_core.lua:121-158, fill 'vgg-mean', scale_factor 1: model_img == nil (in_dim 7, :133-138) or a
        separate image model on pre(img) alone (in_dim 3, :146)."""
        x7 = torch.from_numpy(pyoracle.first_frame_input(content01))[None]
        if self.in_dim == 3:
            x7 = x7[:, :3]
        return self.deprocess(self.forward(x7))[0].to(torch.float64).numpy()

    def run_next_image(self, content01, prev_rgb, flow_lua, cert, warp_mode=0) -> np.ndarray:
        """fast_artistic_video_core.lua:161-180 (+ func_make_last_frame_warped, fast_artistic_video.lua:153-158)."""
        x7 = torch.from_numpy(pyoracle.temporal_input(content01, prev_rgb.astype(np.float32), flow_lua, cert,
                                                      warp_mode=warp_mode))[None]
        return self.deprocess(self.forward(x7))[0].to(torch.float64).numpy()


def make_cert(H, W, idx, use_structure=False, frame=None) -> np.ndarray:
    """Certainty for frame idx exactly as the pipeline produces it: consistencyChecker(bw, fw) -> {0,255} -> /255
    (image.load(pgm,1), fast_artistic_video.lua:103), then utils.min_filter(cert, 7) (core.lua:207)."""
    bw = synth.make_backward_flow(H, W, idx)
    fw = synth.make_forward_flow(H, W, idx)
    img = None
    if use_structure:
        img = np.clip(np.rint(frame * 255.0), 0, 255).astype(np.float32)
    rel = pyoracle.consistency(bw, fw, img)
    cert = rel.astype(np.float32) / 255.0
    return pyoracle.min_filter(cert, 7)


def run_clip(net: NetOracle, H, W, n_frames, warp_mode=0):
    """Frame loop of fast_artistic_video_core.lua:194-229 on the synthetic clip.  Returns list of 3xHxW float64."""
    outs = []
    prev = None
    for i in range(1, n_frames + 1):
        frame = synth.make_frame(H, W, i)
        if i == 1:
            out = net.run_image(frame)
        else:
            cert = make_cert(H, W, i)
            flow = synth.checker_to_lua(synth.make_backward_flow(H, W, i))
            out = net.run_next_image(frame, prev, flow, cert, warp_mode)
        outs.append(out)
        prev = out.astype(np.float32)  # last_frame_stylized = img:clone() (fp32, unclamped), fav.lua:169
    return outs
