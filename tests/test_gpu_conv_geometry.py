"""conv_tc_kernel across the geometries the loss network accepts (csrc/percep.cu), against the fp64 oracle
(oracle/percep_oracle.py).  VGG-16 (test_gpu_percep.py) only reaches 3x3 pad 1 convolutions with 64-channel multiples and
2x2/2 poolings; this sweep runs every wgmma width N = 16 ... 128 (each instance spells out its own accumulator operand
list, wgmma_f16.cuh), Cout below the instance width and partial last N blocks, every plan kind the loss network gets
(tap pairing, 2 or 4 channel blocks per K group, up to 16 K groups, the stride-2 parity split), k 1 / 3 / 5 / 7 with and
without padding, output rows that end 1 pixel into a tile or 1 pixel short of one, padded / ceil / overlapping max-poolings
on either side of the ReLU, and Gram and mean aggregation around one 128-pixel Gram chunk.

Each case is a short chain: a 3 -> Cin convolution (+ ReLU), the convolution under test, then ReLU / max-pooling modules.
Loss layers sit on the tested convolution's own (signed, raw) output and on every module after it."""
import numpy as np
import pytest
import torch

from fav_b200 import percep
from oracle import percep_oracle
from test_gpu_percep import FEATURE_BAR, GRAM_BAR, LOSS_BAR, cuda, images, rel_err

R = dict(type="relu")


def P(k, s, pad=0, ceil=False):
    return dict(type="pool", kW=k, kH=k, dW=s, dH=s, padW=pad, padH=pad, ceil_mode=ceil)


P3x2 = dict(type="pool", kW=3, kH=2, dW=2, dH=1, padW=1, padH=0, ceil_mode=True)  # non-square window, stride and padding


# (cin, cout, k, pad, stride, H, W, modules after the tested conv, aggregation, modules between the first conv and it)
CASES = {
    # every wgmma width, Cout below the instance width
    "n16-cin3-cout1": (3, 1, 3, 1, 1, 5, 129, [R], "gram", None),
    "n16-pair-cout3-k5-ceil": (5, 3, 5, 2, 1, 5, 127, [R, P(2, 2, ceil=True)], "gram", None),
    "n16-cbg2-cout5-k7": (16, 5, 7, 3, 1, 3, 128, [R], "gram", None),
    "n32-cout17-k1": (16, 17, 1, 0, 1, 2, 257, [R], "mean", None),
    "n48-cb6-cout33-pool3s2p1": (48, 33, 3, 1, 1, 5, 128, [R, P(3, 2, 1)], "gram", None),
    "n64-cb6-pad0-pool3s2p1ceil-relu-after": (48, 64, 3, 0, 1, 6, 131, [P(3, 2, 1, True), R], "gram", None),
    "n80-k5pad0-pool2s1": (64, 80, 5, 0, 1, 7, 133, [R, P(2, 1)], "gram", None),
    "n96-cout90-pool3s1p1-relu-after": (64, 90, 3, 1, 1, 4, 127, [P(3, 1, 1), R], "mean", None),
    "n112-cout100-k7": (64, 100, 7, 3, 1, 3, 129, [R], "gram", None),
    "n128-k1": (64, 128, 1, 0, 1, 5, 257, [R], "gram", None),
    # N blocks: 128 + 2 (N 16), 128 + 72 (N 80), 128 + 128 + 44 (N 48)
    "nblk-cin512-cout130-k1": (512, 130, 1, 0, 1, 2, 127, [R], "gram", None),
    "nblk-cout200-ceil-odd": (64, 200, 3, 1, 1, 5, 65, [R, P(2, 2, ceil=True)], "gram", None),
    "nblk-cout300": (16, 300, 3, 1, 1, 4, 96, [R], "mean", None),
    # input channels: 3 and 5 (tap pairing), 16 (CbG 2), 48 (three CbG-2 groups), 64, 512 (16 groups)
    "cin3-k7pad0": (3, 64, 7, 0, 1, 9, 135, [R], "gram", None),
    "cin3-k1": (3, 48, 1, 0, 1, 3, 128, [R], "gram", None),
    "cin5-k1": (5, 32, 1, 0, 1, 3, 128, [R], "gram", None),
    "cin5-k3pad0": (5, 48, 3, 0, 1, 5, 131, [R], "gram", None),
    "cin5-k7": (5, 16, 7, 3, 1, 4, 100, [R], "gram", None),
    "cin16-k5": (16, 64, 5, 2, 1, 4, 100, [R], "gram", None),
    "cin16-k3pad0": (16, 32, 3, 0, 1, 4, 131, [R], "gram", None),
    "cin64-k7pad0": (64, 32, 7, 0, 1, 9, 134, [R], "gram", None),
    "cin512-k3": (512, 128, 3, 1, 1, 3, 129, [R], "gram", None),
    "cin512-k1pad0-n64": (512, 64, 1, 0, 1, 4, 64, [R], "gram", None),
    # stride 2 (k3 pad 1, parity-split operand) on odd and even extents, also after a max-pooling
    "s2-cin16-odd": (16, 32, 3, 1, 2, 9, 257, [R], "gram", None),
    "s2-cin64-even-ceil": (64, 64, 3, 1, 2, 8, 256, [R, P(2, 2, ceil=True)], "gram", None),
    "s2-cin48-n80": (48, 80, 3, 1, 2, 7, 254, [R], "gram", None),
    "s2-cin64-after-pool": (64, 96, 3, 1, 2, 11, 259, [R], "gram", [R, P(3, 2, 1, True)]),
    "s2-cin16-cout200": (16, 200, 3, 1, 2, 5, 131, [R], "mean", None),
    # shapes the stylization net's x-fold plan would take (k >= 5, pad (k-1)/2, Cout <= 4 in a block): generic plan here
    "xfold-shape-16to3-k5": (16, 3, 5, 2, 1, 6, 140, [R], "gram", None),
    "xfold-shape-64to130-k5": (64, 130, 5, 2, 1, 4, 130, [R], "gram", None),
    "xfold-shape-32to4-k7": (32, 4, 7, 3, 1, 5, 140, [R], "gram", None),
    # output widths 1 / 127 / 128 / 129 / 257 with 1 - 5 rows, and images narrower than one tile
    "w1-h5": (64, 64, 3, 1, 1, 5, 1, [R], "gram", None),
    "w1-h1": (16, 17, 3, 1, 1, 1, 1, [R], "mean", None),
    "w127-h1": (64, 96, 3, 1, 1, 1, 127, [R], "gram", None),
    "w128-h2": (16, 80, 3, 1, 1, 2, 128, [R], "gram", None),
    "w40-h3": (64, 112, 3, 1, 1, 3, 40, [R, P(3, 2, 1)], "gram", None),
    # aggregation at C 3 / 17 / 80 / 100 / 200 over 127 / 128 / 129 tap pixels (one Gram chunk is 128 pixels)
    "gram-c3-p127": (16, 3, 3, 1, 1, 1, 127, [R], "gram", None),
    "mean-c3-p128": (5, 3, 3, 1, 1, 2, 64, [R], "mean", None),
    "gram-c17-p128": (16, 17, 3, 1, 1, 2, 64, [R], "gram", None),
    "mean-c17-p129": (16, 17, 3, 1, 1, 3, 43, [R], "mean", None),
    "gram-c80-p129": (64, 80, 3, 1, 1, 1, 129, [R], "gram", None),
    "mean-c80-p127": (64, 80, 3, 1, 1, 1, 127, [R], "mean", None),
    "gram-c100-p128": (64, 100, 3, 1, 1, 4, 32, [R], "gram", None),
    "mean-c100-p129": (64, 100, 3, 1, 1, 3, 43, [R], "mean", None),
    "gram-c200-p129": (64, 200, 3, 1, 1, 3, 43, [R], "gram", None),
    "gram-c200-p127": (64, 200, 3, 1, 1, 1, 127, [R], "gram", None),
    "mean-c200-p128": (64, 200, 3, 1, 1, 2, 64, [R], "mean", None),
    # poolings: non-square (3 wide, 2 tall, strides 2 / 1, padded in x only) at odd extents, and k2 s2 pad 1 ceil at extents
    # 5 and 129, where the last ceil window would start in the padding and is dropped (pool_out)
    "pool-k3x2-s2x1-ceil-odd": (16, 32, 3, 1, 1, 7, 131, [R, P3x2], "gram", None),
    "pool-k2s2p1-ceil-drop": (16, 48, 3, 1, 1, 5, 129, [R, P(2, 2, 1, True)], "gram", None),
    # input channels 32 / 96 / 112 / 192 / 208: the input gradient's wgmma N (32, 96, 112, and 128 + a partial 64 / 80 block)
    "cin32-n16": (32, 16, 3, 1, 1, 4, 128, [R], "gram", None),
    "cin48-k5-pool2s1": (48, 32, 5, 2, 1, 5, 131, [R, P(2, 1)], "gram", None),
    "cin96-k5": (96, 64, 5, 2, 1, 3, 130, [R], "gram", None),
    "cin112-pool3s1p1": (112, 32, 3, 1, 1, 4, 100, [R, P(3, 1, 1)], "gram", None),
    "cin192": (192, 64, 3, 1, 1, 4, 130, [R], "gram", None),
    "cin208-pool2": (208, 32, 3, 1, 1, 3, 129, [R, P(2, 2)], "mean", None),
}


def npads(cout):
    """wgmma N of each 128-channel N block of a convolution (conv_plan.hpp: init_conv_def, conv_nblock_cout)"""
    return [max(16, -(-min(128, cout - b) // 16) * 16) for b in range(0, cout, 128)]


def test_case_table_covers_every_wgmma_width():
    """Trimming the table must not silently drop one of launch_conv_tc's eight instances."""
    widths = {n for case in CASES.values() for n in npads(case[1])}
    assert widths == set(range(16, 129, 16)), sorted(widths)
    assert npads(130) == [128, 16] and npads(300) == [128, 128, 48]


def dgrad_plannable(cin, k):
    """Whether the tensor-core planner runs a stride-1 k x k convolution over `cin` input channels (conv_plan.hpp:
    build_phase_tables): 8 channels (tap pairing), or an even number of 8-channel blocks in K groups of 4 blocks (2 when the
    count is not a multiple of 4), times the filter-row groups that keep one patch stage within 56 KB, at most 16 groups."""
    blocks = -(-cin // 8)
    if blocks == 1:
        return True
    if blocks % 2:
        return False
    cbg = 4 if blocks % 4 == 0 else 2
    nrg = next(rg for rg in range(1, k + 1) if k % rg == 0 and (k // rg) * cbg * (128 + k - 1) * 32 <= 56 * 1024)
    return nrg * (blocks // cbg) <= 16


def backward_refusal(mods):
    """(module index, reason) of the convolution fav_percep_forward_backward refuses, or None: first any stride != 1 or
    pad != (k - 1) / 2, then the first input gradient (a cout -> cin convolution, so Cin = the forward's Cout) without a plan"""
    convs = [(i, m) for i, m in enumerate(mods, 1) if m["type"] == "conv"]
    for i, m in convs:
        if m["stride"] != 1 or m["pad"] != (m["k"] - 1) // 2:
            return i, "stride/pad"
    for i, m in convs:
        if not dgrad_plannable(m["cout"], m["k"]):
            return i, "input gradient"
    return None


def dgrad_widths(name):
    """wgmma N of every input-gradient convolution of a row's chain: N blocks of the forward Cin"""
    mods = chain(name)[0]
    return {n for m in mods if m["type"] == "conv" for n in npads(m["cin"])}


def test_backward_rows_cover_every_input_gradient_width():
    """The rows whose backward runs must reach every wgmma width of the input-gradient convolutions; trimming the table
    must not drop one."""
    runs = [name for name in CASES if backward_refusal(chain(name)[0]) is None]
    widths = set().union(*(dgrad_widths(name) for name in runs))
    assert widths == set(range(16, 129, 16)), sorted(widths)


def test_backward_refusal_rules():
    assert [c for c in (1, 3, 8, 16, 17, 24, 32, 33, 48, 64, 90, 100, 128, 130, 200, 300, 512) if not dgrad_plannable(c, 3)] == \
        [17, 24, 33, 100, 130, 200, 300]
    assert dgrad_plannable(64, 7) and not dgrad_plannable(48, 7) and dgrad_plannable(96, 5) and not dgrad_plannable(128, 5)
    refused = [name for name in CASES if backward_refusal(chain(name)[0])]
    assert len(CASES) - len(refused) == 29 and len(refused) == 26, (len(CASES), len(refused))


def conv(rng, cin, cout, k, pad, stride):
    """He-normal weights as percep.vgg16_modules: activations keep their scale and stay inside the fp16 range"""
    w = rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))
    if cin == 3:
        w /= 128.0  # the preprocessed input spans about +-128
    return dict(type="conv", cin=cin, cout=cout, k=k, stride=stride, pad=pad, weight=w.astype(np.float32),
                bias=(rng.standard_normal(cout) * 0.1).astype(np.float32))


def chain(name):
    cin, cout, k, pad, stride, H, W, post, agg, pre = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    mods = [] if cin == 3 else [conv(rng, 3, cin, 3, 1, 1)] + (pre or [R])
    tested = len(mods) + 1
    mods += [conv(rng, cin, cout, k, pad, stride)] + [dict(m) for m in post]
    return mods, tested, H, W, agg


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_loss_network_geometry_vs_fp64_oracle(name):
    mods, tested, H, W, agg = chain(name)
    layers = list(range(tested, len(mods) + 1))  # the raw conv output and every module after it
    content, cw = [tested, layers[-1]], [1.0, 0.5]
    sw = [1.0 + 0.5 * i for i in range(len(layers))]
    crit = percep.PerceptualCriterion(mods, content, cw, layers, sw, agg_type=agg)
    ora = percep_oracle.PercepOracle(mods, content, cw, layers, sw, agg_type=agg)
    img, stylized, style = images(H, W, 7)
    crit.set_style_target(cuda(style))
    targets = ora.set_style_target(style)
    fstyle = percep_oracle.features(mods, style, layers)
    fmap, aggs = {}, {}
    for k, i in enumerate(layers):
        fmap[f"style f{i}"] = rel_err(crit.layer_output(1, i), fstyle[i], f"style image layer {i}")
        aggs[f"target {i}"] = rel_err(crit.style_stat(0, k), targets[k], f"style target {agg} {i}")
    cl, sl = crit.evaluate(cuda(img), cuda(stylized))
    rc, rs, fc, fs, ref_aggs = ora.evaluate(img, stylized)
    for i in content:
        fmap[f"content f{i}"] = rel_err(crit.layer_output(0, i), fc[i], f"content layer {i}")
    for k, i in enumerate(layers):
        fmap[f"stylized f{i}"] = rel_err(crit.layer_output(1, i), fs[i], f"stylized layer {i}")
        aggs[f"stylized {i}"] = rel_err(crit.style_stat(1, k), ref_aggs[k], f"stylized {agg} {i}")
    ec, es = abs(cl - rc) / abs(rc), abs(sl - rs) / abs(rs)
    print(f"\n{name}: maps {max(fmap.values()):.1e} {agg} {max(aggs.values()):.1e} losses {ec:.1e} {es:.1e}")
    assert max(fmap.values()) <= FEATURE_BAR, fmap
    assert max(aggs.values()) <= GRAM_BAR, aggs
    assert ec <= LOSS_BAR and es <= LOSS_BAR, (cl, rc, sl, rs)
    crit.close()
    torch.cuda.synchronize()
