"""Convolutions with small weights against fp64.  The tensor cores multiply with fp16 pairs hi + lo; a weight below 2^-3 used to
leave lo in the fp16 subnormals, with an absolute error of up to 2^-25 whatever the weight's size, so a conv's relative error
grew as its weights shrank (trained and batch-norm-folded nets sit well below 2^-3).  A conv with max |w| below 2^-6 now packs
its weights times one power of two 2^e that puts max |w| 2^e in [2^14, 2^15) and takes the 2^-e back in the epilogue
(set_weight_prescale, conv_plan.hpp); above, the unscaled split is already within 2^-19 of max |w| and stays as it was.  Here every suite's nets run with their weights times 2^-k, k = 0, 4, 8, 12, against fp64 built from the same
scaled weights, with the bars of the suites they come from; and the worst error at the largest k must stay within 2x of k = 0.
Without the prescale every case below fails its bars or that 2x at its largest k.

The largest k is 12 unless the activations themselves shrink with k to where their own fp16 pairs lose bits (|x| < 2^-3: the
same floor on the activation side, which this file does not test): the loss network's features are stored as fp16 pairs, and
in the paper arch the InstanceNorm of a UX token renormalizes, without a conv to average the errors, an input that the eps of
the InstanceNorm before it has shrunk.  Those cases stop at k = 8, or 4 for a row whose features start near 1.

- Stylization nets: every conv's weight and bias times 2^-k.  InstanceNorm takes the scale out again (until the conv's variance
  falls to its eps, 1e-5), so only the final conv's output shrinks: bounded by 2e-4 max |ref| besides the usual TOL / 10.
- Batch-normalized net: conv weight, bias and running mean times 2^-k, running variance and eps times 4^-k: the same net.
- Loss network: the conv under test of test_gpu_conv_geometry's rows times 2^-k (its input stays the first conv's: scaling that
  one too would shrink the operand itself into the fp16 floor, which is the activation side's precision, not the weights').
  ReLU and max-pooling are positively homogeneous, so the relative bars of the features, Grams and losses still apply."""
import numpy as np
import pytest
import torch

import bn_oracle
import test_gpu_percep_backward as bwd
from fav_b200 import percep, synth
from oracle import percep_oracle
from test_gpu_arch_geometry import ROWS
from test_gpu_batch import WIDE
from test_gpu_conv_geometry import backward_refusal, chain
from test_gpu_net import TOL, T, rand_input
from test_gpu_percep import FEATURE_BAR, GRAM_BAR, LOSS_BAR, cuda, images, rel_err

pytestmark = pytest.mark.gpu

LAYER_BAR = 2e-4  # x max(1, max |ref|) per layer, test_gpu_net.py

# name: ((arch, padding_type, in_dim, H, W), largest k)
NETS = {
    "default-reflect": ((synth.DEFAULT_ARCH, "reflect-start", 7, 64, 96), 12),
    "default-zero": ((synth.DEFAULT_ARCH, "zero", 7, 64, 96), 12),
    "paper": ((synth.PAPER_ARCH, "reflect-start", 7, 64, 96), 8),
    "wide": ((WIDE, "reflect-start", 7, 64, 96), 12),
    "first3-k7-f-s2": (ROWS["first3-k7-f-s2"], 12),
    "xfold-k7-w244": (ROWS["xfold-k7-w244"], 12),
}
# the loss network's conv under test -> largest k: N 16 from 3 channels (tap pairing), N 128, N blocks 128 + 16 and N 64 from
# 512 channels, stride 2
PERCEP_ROWS = {"n16-cin3-cout1": 4, "n128-k1": 8, "nblk-cin512-cout130-k1": 8, "cin512-k1pad0-n64": 8, "s2-cin64-even-ceil": 8}
BACKWARD_ROWS = ["n128-k1", "cin512-k1pad0-n64"]


def is_conv_param(key):
    """'l3.weight', 'l4.c1.bias': a conv's; 'l0.n.weight', 'l4.n2.running_var': a norm's"""
    return key.rsplit(".", 1)[0].split(".")[-1] not in ("n", "n1", "n2")


def scaled(w, k, bn=False):
    out = {}
    for key, v in w.items():
        f = 1.0
        if is_conv_param(key):
            f = 2.0 ** -k
        elif bn and key.endswith(".running_mean"):
            f = 2.0 ** -k
        elif bn and key.endswith((".running_var", ".eps")):
            f = 4.0 ** -k
        out[key] = (v * np.float32(f)).astype(np.float32)
    return out


def net_errors(net, ora, x):
    """(worst layer error / max(1, max |ref|), its layer, net-space output error / 255, output error / max |ref|)"""
    taps = {}
    ref = ora.forward(torch.from_numpy(x)[None], taps)[0].numpy()
    out = net.forward(T(x)[None]).cpu().numpy()[0]
    assert out.shape == ref.shape
    layer = []
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = net.layer_output(i).cpu().numpy()
        assert g.shape == r.shape, (i, g.shape, r.shape)
        layer.append(float(np.abs(g - r).max()) / max(1.0, float(np.abs(r).max())))
    eo = float(np.abs(out - ref).max())
    return max(layer), int(np.argmax(layer)), eo / 255.0, eo / float(np.abs(ref).max())


def check_over_k(name, errors_at, kmax=12):
    """errors_at(k) -> (worst relative error, its bar-checked parts as {what: (value, bar)}); every k = 0, 4, ... kmax within its
    bars, and the worst error at kmax within 2x of k = 0"""
    worst, failed = {}, []
    for k in range(0, kmax + 1, 4):
        worst[k], parts = errors_at(k)
        print(f"  {name} k={k:2d}: worst {worst[k]:.2e}  " + "  ".join(f"{w} {v:.1e}" for w, (v, _) in parts.items()))
        failed += [(k, w, v, bar) for w, (v, bar) in parts.items() if not v <= bar]
    assert not failed, failed
    assert worst[kmax] <= 2 * worst[0], worst


@pytest.mark.parametrize("name", list(NETS))
def test_stylization_net_with_small_weights_vs_fp64(name):
    from fav_b200 import models_video
    from oracle import net_oracle

    (arch, ptype, in_dim, H, W), kmax = NETS[name]
    w0 = synth.make_weights(arch, "scream", in_dim)
    x = rand_input(H, W, 11)[:in_dim]

    def errors_at(k):
        w = scaled(w0, k)
        net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim).load_state(w)
        ora = net_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=w, padding_type=ptype, in_dim=in_dim)
        el, li, eo, er = net_errors(net, ora, x)
        return max(el, er), {f"layer (l{li})": (el, LAYER_BAR), "output/255": (eo, TOL / 10), "output/max": (er, LAYER_BAR)}

    print()
    check_over_k(name, errors_at, kmax)


def test_batch_normalized_net_with_small_weights_vs_fp64():
    from fav_b200 import models_video

    arch, H, W = synth.DEFAULT_ARCH, 64, 96
    w0 = bn_oracle.calibrate_bn_weights(arch, "candy", 7, H, W)
    x = bn_oracle.calibration_input(H, W, seed=9)

    def errors_at(k):
        w = scaled(w0, k, bn=True)
        net = models_video.StyleNet(arch, norm="batch").load_state(w)
        ora = bn_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=w)
        el, li, eo, er = net_errors(net, ora, x)
        return max(el, er), {f"layer (l{li})": (el, LAYER_BAR), "output/255": (eo, TOL / 10), "output/max": (er, LAYER_BAR)}

    print()
    check_over_k("batch norm", errors_at)


def scaled_chain(name, k):
    mods, tested, H, W, agg = chain(name)
    m = mods[tested - 1]
    m["weight"] = (m["weight"] * np.float32(2.0 ** -k)).astype(np.float32)
    m["bias"] = (m["bias"] * np.float32(2.0 ** -k)).astype(np.float32)
    return mods, tested, H, W, agg


@pytest.mark.parametrize("name", list(PERCEP_ROWS))
def test_loss_network_with_small_weights_vs_fp64(name):
    """test_gpu_conv_geometry's check of one row, at each k: features, Gram / mean statistics and losses, relative"""

    def errors_at(k):
        mods, tested, H, W, agg = scaled_chain(name, k)
        layers = list(range(tested, len(mods) + 1))
        content, cw = [tested, layers[-1]], [1.0, 0.5]
        sw = [1.0 + 0.5 * i for i in range(len(layers))]
        crit = percep.PerceptualCriterion(mods, content, cw, layers, sw, agg_type=agg)
        ora = percep_oracle.PercepOracle(mods, content, cw, layers, sw, agg_type=agg)
        img, stylized, style = images(H, W, 7)
        crit.set_style_target(cuda(style))
        targets = ora.set_style_target(style)
        fstyle = percep_oracle.features(mods, style, layers)
        fmap, aggs = [], []
        for j, i in enumerate(layers):
            fmap.append(rel_err(crit.layer_output(1, i), fstyle[i], f"style image layer {i}"))
            aggs.append(rel_err(crit.style_stat(0, j), targets[j], f"style target {agg} {i}"))
        cl, sl = crit.evaluate(cuda(img), cuda(stylized))
        rc, rs, fc, fs, ref_aggs = ora.evaluate(img, stylized)
        fmap += [rel_err(crit.layer_output(0, i), fc[i], f"content layer {i}") for i in content]
        for j, i in enumerate(layers):
            fmap.append(rel_err(crit.layer_output(1, i), fs[i], f"stylized layer {i}"))
            aggs.append(rel_err(crit.style_stat(1, j), ref_aggs[j], f"stylized {agg} {i}"))
        crit.close()
        torch.cuda.synchronize()
        ec, es = abs(cl - rc) / abs(rc), abs(sl - rs) / abs(rs)
        parts = {"features": (max(fmap), FEATURE_BAR), agg: (max(aggs), GRAM_BAR), "content loss": (ec, LOSS_BAR),
                 "style loss": (es, LOSS_BAR)}
        return max(v for v, _ in parts.values()), parts

    print()
    check_over_k(name, errors_at, PERCEP_ROWS[name])


@pytest.mark.parametrize("name", BACKWARD_ROWS)
def test_loss_network_backward_with_small_weights_vs_fp64(name):
    """test_gpu_percep_backward's per-pixel gradient check of one row with the conv under test times 2^-8: its input gradient
    runs the transposed, flipped weights through conv_tc_kernel with their own power of two"""
    mods, tested, H, W, agg = scaled_chain(name, 8)
    assert backward_refusal(mods) is None
    cl, cw, sl, sw = bwd.geometry_layers(mods, tested)
    content, stylized, style = bwd.images(H, W, 7)
    crit, targets = bwd.setup(mods, cl, cw, sl, sw, agg, style)
    x, xc = bwd.net_space(stylized), bwd.net_space(content)
    grad, tc, ts, lay = bwd.run(crit, x, xc)
    print()
    _, per = bwd.check_backward(crit, mods, grad, x, xc, cl, cw, sl, sw, targets, agg, f"{name} k=8")
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    assert max(lay_e) <= bwd.LOSS_BAR, lay_e
    crit.close()
