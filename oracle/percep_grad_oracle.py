"""fp64 reference for the gradient of fav_percep_forward_backward (csrc/percep.cu) that takes the GPU's discrete decisions.

The gradient of the loss network jumps where a ReLU's input or a max-pooling window's two largest values lie within rounding
of each other: either side is right, and one such unit moves the gradient of its whole receptive field.  The backward pass
reads its decisions from the fp32 conv outputs it keeps (fav_percep_conv_output): the ReLU mask `raw > 0` and, per pooling
window, the first strict maximum of `raw` in row-major order (padding cells excluded).  This module runs the same module
chain in fp64 with those decisions fixed -- ReLU as `z * M`, max-pooling as a gather at the given arg-max -- so what is left
is a linear map of continuous values, and fp64 autograd of it can be compared with the GPU at every pixel.

`modules` are the dicts of percep_oracle (conv / relu / pool).  Without `raws` every decision is the fp64 forward's own, and
the gradient equals plain autograd through torch.relu / F.max_pool2d."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def pool_out(n, k, s, p, ceil_mode):
    """SpatialMaxPooling's output extent (THNN): floor or ceil, then 'the last window starts inside the image' when padded"""
    o = (math.ceil if ceil_mode else math.floor)((n - k + 2 * p) / s) + 1
    if p > 0 and (o - 1) * s >= n + p:
        o -= 1
    return o


def pool_argmax(d, m):
    """d [C,H,W] -> [C,Ho,Wo] flat indices (y * W + x) of each window's first strict maximum in row-major order, padding
    cells excluded; the windows of pool module m"""
    C, H, W = d.shape
    kH, kW, dH, dW, pH, pW = m["kH"], m["kW"], m["dH"], m["dW"], m["padH"], m["padW"]
    Ho, Wo = pool_out(H, kH, dH, pH, m["ceil_mode"]), pool_out(W, kW, dW, pW, m["ceil_mode"])
    bottom = max(0, (Ho - 1) * dH + kH - pH - H)
    right = max(0, (Wo - 1) * dW + kW - pW - W)
    dp = F.pad(d.detach(), (pW, right, pH, bottom), value=-math.inf)
    win = dp.unfold(1, kH, dH).unfold(2, kW, dW)[:, :Ho, :Wo].reshape(C, Ho, Wo, kH * kW)
    # the first maximum: the largest value, then the smallest window position among the cells that hold it
    top = win.max(-1, keepdim=True).values
    pos = torch.arange(kH * kW, device=d.device).expand_as(win)
    j = torch.where(win == top, pos, kH * kW).min(-1).values
    oy = torch.arange(Ho, device=d.device)[:, None] * dH - pH
    ox = torch.arange(Wo, device=d.device)[None, :] * dW - pW
    return (oy + torch.div(j, kW, rounding_mode="floor")) * W + ox + j % kW


def gather(z, idx):
    C = z.shape[0]
    return z.reshape(C, -1).gather(1, idx.reshape(C, -1)).reshape(idx.shape)


def _weights(m, dev):
    return (torch.as_tensor(np.asarray(m["weight"], np.float64), device=dev),
            torch.as_tensor(np.asarray(m["bias"], np.float64), device=dev))


def features(mods, x, indices, raws=None, decisions=None):
    """{index: [C,H,W]} of the chain from a net-space [3,H,W] fp64 tensor (differentiable), with every ReLU and max-pooling
    decided by `raws` ({conv module index: its GPU fp32 output [C,H,W]}), or by the chain's own values when raws is None.

    decisions: a list that receives, per ReLU / pooling module where raws is given, (module index, kind, n, worst): the units
    whose decision differs from the fp64 forward's own, and the largest of |z| (ReLU: the fp64 pre-activation) or of the fp64
    gap between the window's maximum and the value at the GPU's arg-max (pooling), over max |z| of the stage's conv output."""
    want, out = set(indices), {}
    z = x
    d = d64 = None  # the values the decisions are read from: the GPU's, and the fp64 forward's own
    zmax = 1.0
    for i, m in enumerate(mods[:max(want)], 1):
        if m["type"] == "conv":
            w, b = _weights(m, x.device)
            z = F.conv2d(z[None], w, b, stride=m["stride"], padding=m["pad"])[0]
            d64 = z.detach()
            d = d64 if raws is None else raws[i].to(x.device, torch.float64)
            assert d.shape == z.shape, (i, d.shape, z.shape)
            zmax = float(d64.abs().max()) or 1.0
        elif m["type"] == "relu":
            mask = d > 0
            if raws is not None and decisions is not None:
                diff = mask != (d64 > 0)
                n = int(diff.sum())
                decisions.append((i, "relu", n, float(d64[diff].abs().max()) / zmax if n else 0.0))
            z = z * mask
        else:
            idx = pool_argmax(d, m)
            if raws is not None and decisions is not None:
                own = pool_argmax(d64, m)
                diff = idx != own
                n = int(diff.sum())
                gap = (gather(d64, own) - gather(d64, idx))[diff]
                decisions.append((i, "pool", n, float(gap.abs().max()) / zmax if n else 0.0))
                d64 = gather(d64, own)
            else:
                d64 = gather(d64, idx)
            z, d = gather(z, idx), gather(d, idx)
        if i in want:
            out[i] = z
    return out


def plain_features(mods, x, indices):
    """{index: [C,H,W]} through torch.relu and F.max_pool2d themselves (differentiable)"""
    want, out = set(indices), {}
    z = x[None]
    for i, m in enumerate(mods[:max(want)], 1):
        if m["type"] == "conv":
            w, b = _weights(m, x.device)
            z = F.conv2d(z, w, b, stride=m["stride"], padding=m["pad"])
        elif m["type"] == "relu":
            z = torch.relu(z)
        else:
            z = F.max_pool2d(z, (m["kH"], m["kW"]), (m["dH"], m["dW"]), (m["padH"], m["padW"]), ceil_mode=bool(m["ceil_mode"]))
        if i in want:
            out[i] = z[0]
    return out


def aggregate(f, agg_type):
    C, H, W = f.shape
    x = f.reshape(C, H * W)
    return x @ x.t() / (C * H * W) if agg_type == "gram" else x.mean(1)


def grad(mods, x, xc, cl, cw, sl, sw, targets, agg_type, raws=None, device="cpu", plain=False):
    """d PerceptualCriterion / d x for the net-space input x [3,H,W] (content target xc) in fp64.

    Returns (grad [3,H,W] fp64 cpu, per-layer losses (content layers, then style layers), decisions (see features)).
    The content features of xc and the style targets (`targets`, percep_oracle.PercepOracle.set_style_target) are plain fp64;
    plain=True runs the chain through torch.relu / F.max_pool2d instead of fixed decisions."""
    X = torch.as_tensor(x).to(device, torch.float64).requires_grad_()
    layers = list(cl) + list(sl)
    decisions = []
    with torch.no_grad():
        fc = plain_features(mods, torch.as_tensor(xc).to(device, torch.float64), cl) if cl else {}
    fs = plain_features(mods, X, layers) if plain else features(mods, X, layers, raws, decisions)
    per = [w * ((fs[i] - fc[i]) ** 2).mean() for i, w in zip(cl, cw)]
    per += [w * ((aggregate(fs[i], agg_type) - torch.as_tensor(t).to(device, torch.float64)) ** 2).mean()
            for i, w, t in zip(sl, sw, targets)]
    (g,) = torch.autograd.grad(sum(per), X)
    return g.cpu(), [float(v.detach()) for v in per], decisions


PIXEL_BAR = 1e-3   # max |got - ref| <= PIXEL_BAR * max |ref|, over the whole gradient and over its outer two rows and columns


def pixel_err(got, ref, border=2):
    """(max |got - ref| / max |ref|, the same over the outer `border` rows and columns against their own max |ref|)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    d = np.abs(got - ref)
    edge = np.zeros(ref.shape[-2:], bool)
    edge[:border], edge[-border:], edge[:, :border], edge[:, -border:] = True, True, True, True
    m, me = float(np.abs(ref).max()), float(np.abs(ref[..., edge]).max())
    return float(d.max()) / m if m else float(d.max()), float(d[..., edge].max()) / me if me else float(d[..., edge].max())

