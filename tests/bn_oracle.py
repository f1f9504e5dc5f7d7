"""fp64 restatement of batch-normalized stylization nets (-use_instance_norm 0).  TEST INFRASTRUCTURE ONLY.

models_video.lua:21-25,33-37,121-127 put nn.SpatialBatchNormalization wherever the default has InstanceNormalization, and
get_model evaluates the net (fast_artistic_video_core.lua:46): each BN is F.batch_norm(training=False) with its running
statistics.  Everything else is oracle.net_oracle.NetOracle.

No trained BN checkpoint exists here, so calibrate_bn_weights gives the running statistics a trained net would have: the
per-channel mean and variance of each BN's input on a seeded frame, taken layer by layer, then perturbed (mean +- 0.1 std,
variance x 0.7-1.4) so that the BN is not an InstanceNorm in disguise.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from fav_b200 import synth
from oracle import net_oracle, pyoracle


class NetOracle(net_oracle.NetOracle):
    """net_oracle.NetOracle with norm='batch': inference-mode SpatialBatchNormalization; weights need the '<n>.running_mean',
    '<n>.running_var' and '<n>.eps' entries of synth.make_weights(norm='batch').  `hook(name, x)`, if given, is called with each
    BN's input before it is applied (calibrate_bn_weights)."""

    def __init__(self, *args, norm="batch", hook=None, **kw):
        assert norm == "batch"
        super().__init__(*args, **kw)
        self.hook = hook

    def _bn(self, x, name):
        if self.hook is not None:
            self.hook(name, x)
        w = self.w
        return F.batch_norm(x, w[name + ".running_mean"], w[name + ".running_var"], w[name + ".weight"], w[name + ".bias"],
                            training=False, eps=float(w[name + ".eps"].reshape(-1)[0]))

    def forward(self, x7, taps=None):
        x = x7.to(self.dtype)
        if self.pad:
            x = F.pad(x, (self.pad,) * 4, mode="reflect")  # train_video.lua:322
        for i, s in enumerate(self.specs):
            n = f"l{i}"
            if s["kind"] == "conv":
                x = self._conv(x, n, s["stride"], s["pad"])
            elif s["kind"] == "fullconv":
                x = self._fullconv(x, n, s)
            elif s["kind"] == "up":
                x = F.interpolate(x, scale_factor=s["scale"], mode="nearest")
            elif s["kind"] == "res":  # build_conv_block :10-39 (+ ConcatTable / CAddTable :41-53 for RX)
                bp = self.block_pad
                y = self._conv(x, n + ".c1", 1, bp)
                y = torch.relu(self._bn(y, n + ".n1"))
                y = self._conv(y, n + ".c2", 1, bp)
                y = self._bn(y, n + ".n2")
                if not s.get("skip", True):
                    x = y
                elif bp:
                    x = y + x
                else:
                    x = y + x[:, :, 2:-2, 2:-2]
            if s["in_norm"]:
                x = self._bn(x, n + ".n")
            if s["relu"]:
                x = torch.relu(x)
            if taps is not None:
                taps[n] = x
        return torch.tanh(x) * self.tanh_constant


def calibration_input(H, W, in_dim=7, seed=0):
    """A seeded net input: preprocessed frame 1, a random warped previous frame and a random certainty."""
    rng = np.random.default_rng(seed)
    x7 = pyoracle.first_frame_input(synth.make_frame(H, W, 1))
    x7[3:6] = rng.normal(0, 50, (3, H, W))
    x7[6] = rng.uniform(0, 1, (H, W))
    return x7[:in_dim].astype(np.float32)


def calibrate_bn_weights(arch=synth.DEFAULT_ARCH, style="candy", in_dim=7, H=64, W=96, padding_type="reflect-start", seed=0):
    """synth.make_weights(norm='batch') with each BN's running statistics set, in execution order, from the statistics of its
    input on calibration_input(H, W): mean + 0.1 std U(-1, 1), variance x U(0.7, 1.4) (seeded)."""
    w = synth.make_weights(arch, style, in_dim, norm="batch")
    rng = np.random.default_rng(synth.style_seed(style) + 1)

    def hook(name, x):
        m = x.mean(dim=(0, 2, 3)).numpy()
        v = x.var(dim=(0, 2, 3), unbiased=False).numpy()
        c = m.size
        w[name + ".running_mean"] = (m + 0.1 * np.sqrt(v) * rng.uniform(-1, 1, c)).astype(np.float32)
        w[name + ".running_var"] = (v * rng.uniform(0.7, 1.4, c)).astype(np.float32)
        ora.w[name + ".running_mean"] = torch.from_numpy(w[name + ".running_mean"]).double()
        ora.w[name + ".running_var"] = torch.from_numpy(w[name + ".running_var"]).double()

    ora = NetOracle(arch=arch, dtype=torch.float64, weights=w, in_dim=in_dim, padding_type=padding_type, hook=hook)
    ora.forward(torch.from_numpy(calibration_input(H, W, in_dim, seed))[None])
    return w
