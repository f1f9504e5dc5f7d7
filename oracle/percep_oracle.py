"""fp64 PyTorch-CPU restatement of nn.PerceptualCriterion for -evaluate (fast_artistic_video/PerceptualCriterion.lua:27-155,
ContentLoss.lua:39-48, StyleLoss.lua:39-55, GramMatrix.lua:31-53, preprocess.lua:57-62) -- the test oracle of csrc/percep.cu.

`modules` are the dicts of fav_b200.t7.loss_network_from_model: conv (F.conv2d + bias), relu, pool (F.max_pool2d with the
module's kernel / stride / padding / ceil_mode).  The feature map of a layer index is the output of that top-level module."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

VGG_MEAN_BGR = (103.939, 116.779, 123.68)


def preprocess(rgb: np.ndarray) -> torch.Tensor:
    """preprocess.vgg.preprocess on one [3,H,W] image in [0,1]: BGR, x255, minus the mean (fp64)."""
    x = torch.from_numpy(np.asarray(rgb, np.float64))[[2, 1, 0]] * 255.0
    return (x - torch.tensor(VGG_MEAN_BGR, dtype=torch.float64)[:, None, None])[None]


def features(modules, rgb: np.ndarray, indices) -> dict:
    """{index: [C,H,W] fp64 tensor} for every requested (1-based) module index."""
    want = set(indices)
    x = preprocess(rgb)
    out = {}
    for i, m in enumerate(modules[:max(want)], 1):
        if m["type"] == "conv":
            w = torch.from_numpy(np.asarray(m["weight"], np.float64))
            b = torch.from_numpy(np.asarray(m["bias"], np.float64))
            x = F.conv2d(x, w, b, stride=m["stride"], padding=m["pad"])
        elif m["type"] == "relu":
            x = torch.relu(x)
        else:
            x = F.max_pool2d(x, (m["kH"], m["kW"]), (m["dH"], m["dW"]), (m["padH"], m["padW"]), ceil_mode=bool(m["ceil_mode"]))
        if i in want:
            out[i] = x[0].clone()
    return out


def aggregate(f: torch.Tensor, agg_type: str = "gram") -> torch.Tensor:
    """GramMatrix (F F^T / (C H W)) or the per-channel spatial mean of two nn.Mean."""
    C, H, W = f.shape
    x = f.reshape(C, H * W)
    if agg_type == "gram":
        return x @ x.t() / (C * H * W)
    return x.mean(1)


def mse(a: torch.Tensor, b: torch.Tensor) -> float:
    """nn.MSECriterion (sizeAverage): mean over every element."""
    return float(((a - b) ** 2).mean())


class PercepOracle:
    def __init__(self, modules, content_layers, content_weights, style_layers, style_weights, agg_type="gram"):
        self.modules = modules
        self.cl, self.cw = [int(v) for v in content_layers], [float(v) for v in content_weights]
        self.sl, self.sw = [int(v) for v in style_layers], [float(v) for v in style_weights]
        self.agg_type = agg_type
        self.targets = None

    def set_style_target(self, style_rgb):
        f = features(self.modules, style_rgb, self.sl)
        self.targets = [aggregate(f[i], self.agg_type) for i in self.sl]
        return self.targets

    def evaluate(self, content_rgb, stylized_rgb):
        """(total_content_loss, total_style_loss, content features, stylized features, stylized aggregates)"""
        fc = features(self.modules, content_rgb, self.cl)
        fs = features(self.modules, stylized_rgb, self.cl + self.sl)
        content = sum(w * mse(fs[i], fc[i]) for i, w in zip(self.cl, self.cw))
        aggs = [aggregate(fs[i], self.agg_type) for i in self.sl]
        style = sum(w * mse(a, t) for a, t, w in zip(aggs, self.targets, self.sw))
        return content, style, fc, fs, aggs
