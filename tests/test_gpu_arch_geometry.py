"""The stylization net at every geometry an arch token can give it (models_video.lua:55-140), against the fp64 oracle, every
layer.  test_gpu_net.py runs the released archs and a few more tokens; this table adds the first (tap-paired) conv at k 1 / 3 /
5 / 7 from 7 and from 3 channels, non-final 1x1 / 5x5 / 7x7 / 9x9 convs, the x-fold final conv at k 7 (tile stride 122, also
from 16 channels) and at the tile edges of k 5 and 7, the generic and tap-paired final convs, stride-1 transposed convs at
k 1 / 5 / 7 / 9 (flipped filter, zero border tpad up to 4), stride-2 transposed convs at k 7 / 9 (sub-pixel phases with
16/12/12/9 and 25/20/20/16 taps), nearest upsampling by 1 and 4, residual and conv blocks at two scales in both padding
types, and three stride-2 layers.  Bars as test_gpu_net.py: 2e-4 * max(1, max|ref|) per layer, TOL / 10 on the net-space
output / 255 and on run_image, 5e-5 between the tensor-core path and the CUDA-core comparator."""
import functools

import numpy as np
import pytest
import torch

from fav_b200 import synth
from test_gpu_net import TOL, T, rand_input

pytestmark = pytest.mark.gpu

THREE_S2 = "c9s1-32,d64,d128,d128,R128,u128,u64,u32,c9s1-3"

# name: (arch, padding_type, in_dim, H, W)
ROWS = {
    # first conv from 7 channels (tap pairing) k 1; generic final c1s1-3
    "first7-k1": ("c1s1-32,d64,R64,u32,c1s1-3", "reflect-start", 7, 64, 96),
    # first conv k 3; x-fold final c7s1-3 from 32 (N = 7 x 3 -> 32, tile stride 122)
    "first7-k3": ("c3s1-32,d64,R64,u32,c7s1-3", "reflect-start", 7, 64, 96),
    # first conv k 5; x-fold final c7s1-3 from 16 (CbG 2)
    "first7-k5": ("c5s1-32,d64,R64,u16,c7s1-3", "reflect-start", 7, 64, 96),
    # first conv k 7; non-final c9s1 from 16, c5s1 from 32 (223 KB of shared memory), c5s1 / c7s1 / c1s1 from 64
    "first7-k7-nonfinal": ("c7s1-16,c9s1-32,c5s1-32,d64,c5s1-64,c7s1-64,c1s1-64,R64,u32,c9s1-3", "reflect-start", 7, 64, 96),
    # first conv from 3 channels k 1; non-final c1s1 from 128; x-fold c5s1-3
    "first3-k1": ("c1s1-32,d64,d128,c1s1-128,R128,u64,u32,c5s1-3", "reflect-start", 3, 64, 96),
    # first conv from 3 channels k 3; final c5s1-3 from 8 channels (tap pairing, plain final epilogue)
    "first3-k3": ("c3s1-32,d64,R64,u8,c5s1-3", "reflect-start", 3, 64, 96),
    # first conv from 3 channels k 5; stride-1 transposed convs f1s1 / f5s1 / f7s1 / f9s1 (tpad 0 / 2 / 3 / 4)
    "first3-k5-f-s1": ("c5s1-32,d64,f1s1-64,f5s1-64,f7s1-64,f9s1-32,u16,c9s1-3", "reflect-start", 3, 64, 96),
    # first conv from 3 channels k 7; stride-2 transposed f7s2 from 128 and f9s2 from 64 (tpad 1 and 2)
    "first3-k7-f-s2": ("c7s1-32,d64,d128,R128,f7s2-64,f9s2-32,c9s1-3", "reflect-start", 3, 64, 96),
    # nearest upsampling by 4 (up_apply on 128 channels); x-fold c9s1-3 from 128
    "U4": ("c9s1-32,d64,d128,R128,U4,c9s1-3", "reflect-start", 7, 64, 96),
    # nearest upsampling by 1: InstanceNorm + ReLU only
    "U1": ("c9s1-32,d64,U1,R64,u32,c9s1-3", "reflect-start", 7, 64, 96),
    # residual and conv blocks at full and half resolution; reflect-start pad 4 + 8 + 8 + 4 = 24, halved to 12
    "blocks-mixed-reflect": ("c9s1-32,R32,d64,C64,R64,u32,R32,c9s1-3", "reflect-start", 7, 64, 96),
    "blocks-mixed-zero": ("c9s1-32,R32,d64,C64,R64,u32,R32,c9s1-3", "zero", 7, 64, 96),
    # three stride-2 layers at a size they restore (multiples of 8)
    "three-s2": (THREE_S2, "reflect-start", 7, 72, 104),
    # x-fold tile edges: k 5 strides 124 pixels (W 248 = 2 tiles, 252 = 2 tiles + 4), k 7 strides 122 (244 / 248)
    "xfold-k5-w248": ("c9s1-32,d64,R64,u32,c5s1-3", "reflect-start", 7, 32, 248),
    "xfold-k5-w252": ("c9s1-32,d64,R64,u32,c5s1-3", "reflect-start", 7, 32, 252),
    "xfold-k7-w244": ("c9s1-32,d64,R64,u32,c7s1-3", "reflect-start", 7, 32, 244),
    "xfold-k7-w248": ("c9s1-32,d64,R64,u32,c7s1-3", "reflect-start", 7, 32, 248),
}

# batch-normalized: operand epilogues writing consumers with padT 3 / 4 (c7s1, c9s1) and tpad 2 - 4 (f5s1 / f7s1 / f9s1)
BN_ROWS = ["first7-k7-nonfinal", "first3-k5-f-s1"]
BATCH_ROW = "first3-k7-f-s2"  # sub-pixel phases of every image in one launch


def make_net(name, norm="instance"):
    from fav_b200 import models_video
    from oracle import net_oracle

    arch, ptype, in_dim, H, W = ROWS[name]
    if norm == "batch":
        import bn_oracle

        w = bn_oracle.calibrate_bn_weights(arch, "candy", in_dim, H, W, padding_type=ptype)
        ora = bn_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=w, padding_type=ptype, in_dim=in_dim)
    else:
        w = synth.make_weights(arch, "scream", in_dim)
        ora = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=in_dim)
    net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim, norm=norm).load_state(w)
    return net, ora


def net_input(name, seed):
    _, _, in_dim, H, W = ROWS[name]
    return rand_input(H, W, seed)[:in_dim]


def check_vs_oracle(name, net, ora, x):
    """Every layer, the net-space output and run_image against the oracle; returns the worst errors (per layer relative to
    max(1, max|ref|), output / 255, run_image)."""
    _, _, _, H, W = ROWS[name]
    taps = {}
    ref = ora.forward(torch.from_numpy(x)[None], taps)[0].numpy()
    out = net.forward(T(x)[None]).cpu().numpy()[0]
    assert out.shape == ref.shape == (3, H, W)
    layer = []
    for i in range(len(ora.specs) - 1):
        r = taps[f"l{i}"][0].numpy()
        g = net.layer_output(i).cpu().numpy()
        assert g.shape == r.shape, (i, g.shape, r.shape)
        layer.append(np.abs(g - r).max() / max(1.0, np.abs(r).max()))
    worst = int(np.argmax(layer))
    assert layer[worst] < 2e-4, f"layer {worst}: {layer}"
    eo = np.abs(out - ref).max() / 255.0
    assert eo < TOL / 10, eo
    f1 = synth.make_frame(H, W, 1)
    er = np.abs(net.run_image(T(f1)).cpu().numpy() - ora.run_image(f1)).max()
    assert er < TOL / 10, er
    return layer[worst], worst, eo, er


def simt_agreement(net, x):
    xt = T(x)[None]
    a = net.forward(xt)
    net.set_conv_impl("simt")
    try:
        b = net.forward(xt)
    finally:
        net.set_conv_impl("tcgen05")
    return float((a - b).abs().max()) / 255.0


@pytest.mark.parametrize("name", list(ROWS))
def test_arch_geometry_every_layer_vs_fp64_oracle(name):
    net, ora = make_net(name)
    x = net_input(name, 11)
    el, worst, eo, er = check_vs_oracle(name, net, ora, x)
    es = simt_agreement(net, x)
    print(f"\n{name}: worst layer {el:.1e} (l{worst}) output {eo:.1e} run_image {er:.1e} vs CUDA cores {es:.1e}")
    assert es < 5e-5, es


@pytest.mark.parametrize("name", BN_ROWS)
def test_bn_arch_geometry_every_layer_vs_fp64_oracle(name):
    import bn_oracle

    net, ora = make_net(name, norm="batch")
    _, _, in_dim, H, W = ROWS[name]
    x = bn_oracle.calibration_input(H, W, in_dim, seed=9)
    el, worst, eo, er = check_vs_oracle(name, net, ora, x)
    es = simt_agreement(net, x)
    print(f"\n{name} (batch norm): worst layer {el:.1e} (l{worst}) output {eo:.1e} run_image {er:.1e} vs CUDA cores {es:.1e}")
    assert es < 5e-5, es


def test_batch_of_three_is_each_image_alone():
    net, _ = make_net(BATCH_ROW)
    xs = [net_input(BATCH_ROW, 20 + b) for b in range(3)]
    n_layers = len(synth.parse_arch(ROWS[BATCH_ROW][0])) - 1
    alone = []
    for x in xs:
        out = net.forward(T(x)[None])[0].cpu()
        alone.append((out, [net.layer_output(i).cpu() for i in range(n_layers)]))
    out = net.forward(T(np.stack(xs))).cpu()
    for b, (o, taps) in enumerate(alone):
        assert torch.equal(out[b], o), f"image {b}"
        for i in range(n_layers):
            assert torch.equal(net.layer_output(i, b).cpu(), taps[i]), f"image {b}, layer {i}"


def test_c3s2_tokens_are_d_tokens():
    """cXsY-Z with X 3, Y 2 builds SpatialConvolution(3,3,2,2,1,1) (models_video.lua:65-80), the conv a dZ token builds (:90-93):
    with the same weights the two archs are the same net."""
    from fav_b200 import models_video

    arch = "c9s1-32,c3s2-64,c3s2-128,R128,R128,R128,R128,R128,u64,u32,c9s1-3"
    w = synth.make_weights(synth.DEFAULT_ARCH, "candy")
    alt = synth.make_weights(arch, "candy")
    assert sorted(alt) == sorted(w) and all(np.array_equal(alt[k], w[k]) for k in w)
    a = models_video.StyleNet(synth.DEFAULT_ARCH).load_state(w)
    b = models_video.StyleNet(arch).load_state(w)
    x = T(rand_input(64, 96, 4))[None]
    assert torch.equal(a.forward(x), b.forward(x))
    f1 = T(synth.make_frame(64, 96, 1))
    assert torch.equal(a.run_image(f1), b.run_image(f1))


@pytest.mark.parametrize("shape", [(68, 68), (72, 100)])
def test_frame_sizes_the_arch_does_not_restore_are_refused(shape):
    """Three stride-2 layers restore a frame whose sides are multiples of 8: at 68x68 the net would return 72x72 (see
    test_arch_geometry_tables.py), at 72x100 a 72x104 frame.  forward and run_image refuse both sizes before any kernel runs;
    the net still runs a size it restores afterwards."""
    from fav_b200 import _lib, models_video

    H, W = shape
    net = models_video.StyleNet(THREE_S2).load_state(synth.make_weights(THREE_S2, "scream"))
    with pytest.raises(_lib.FavError) as e:
        net.forward(torch.zeros((1, 7, H, W), device="cuda"))
    assert e.value.status == _lib.FAV_ERR_INVALID and "multiples of 8" in str(e.value), str(e.value)
    with pytest.raises(_lib.FavError) as e:
        net.run_image(torch.zeros((3, H, W), device="cuda"))
    assert e.value.status == _lib.FAV_ERR_INVALID
    out = net.run_image(T(synth.make_frame(72, 104, 1)))
    assert out.shape == (3, 72, 104) and bool(torch.isfinite(out).all())
