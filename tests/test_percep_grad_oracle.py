"""The fixed-decision fp64 reference of the loss network's backward pass (oracle/percep_grad_oracle.py), on the CPU: it equals
plain autograd when it takes the fp64 forward's own decisions, its arg-max is the first strict maximum of every window, and the
per-pixel bar it makes possible catches wrong gradients that the statistical bar (99th percentile and relative L2) lets pass."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fav_b200 import percep
from oracle import percep_grad_oracle as pgo
from oracle import percep_oracle
from test_gpu_conv_geometry import CASES, P3x2, backward_refusal, chain
from test_gpu_percep import images

OLD_BAR = 2e-2  # the statistical bar: 99th percentile of |got - ref| / max |ref| and relative L2 error
BACKWARD_ROWS = [name for name in CASES if backward_refusal(chain(name)[0]) is None]
MEAN_BGR = torch.tensor(percep_oracle.VGG_MEAN_BGR, dtype=torch.float64)[:, None, None]


def net_space(rgb):
    return torch.from_numpy(np.asarray(rgb, np.float64))[[2, 1, 0]] * 255.0 - MEAN_BGR


def layer_setup(mods, tested, agg):
    """the loss layers of test_gpu_conv_geometry: the tested conv's raw output and every module after it, content on the
    first and the last; style targets from the style image"""
    layers = list(range(tested, len(mods) + 1))
    cl, cw = [tested, layers[-1]], [1.0, 0.5]
    sw = [1.0 + 0.5 * i for i in range(len(layers))]
    return cl, cw, layers, sw


def targets_of(mods, sl, sw, agg, style):
    return percep_oracle.PercepOracle(mods, [], [], sl, sw, agg).set_style_target(style) if sl else []


def max_rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


@pytest.mark.parametrize("name", BACKWARD_ROWS)
def test_own_decisions_equal_plain_autograd(name):
    mods, tested, H, W, agg = chain(name)
    W = min(W, 40)
    cl, cw, sl, sw = layer_setup(mods, tested, agg)
    content, stylized, style = images(H, W, 7)
    x, xc = net_space(stylized), net_space(content)
    targets = targets_of(mods, sl, sw, agg, style)
    g, per, dec = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, agg)
    gp, perp, _ = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, agg, plain=True)
    assert dec == []
    assert float(gp.abs().max()) > 0
    assert max_rel(g, gp) <= 1e-12, max_rel(g, gp)
    assert all(abs(a - b) <= 1e-12 * abs(b) for a, b in zip(per, perp)), (per, perp)


def test_own_decisions_equal_plain_autograd_vgg16_pool3():
    mods = percep.vgg16_modules(18)
    for m in mods:
        if m["type"] == "pool":
            m.update(kW=3, kH=3, dW=2, dH=2, padW=1, padH=1, ceil_mode=True)
    content, stylized, style = images(34, 46, 3)
    x, xc = net_space(stylized), net_space(content)
    cl, cw, sl, sw = [10], [1.0], [5, 16], [1.0, 2.0]
    targets = targets_of(mods, sl, sw, "gram", style)
    g, _, _ = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, "gram")
    gp, _, _ = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, "gram", plain=True)
    assert max_rel(g, gp) <= 1e-12, max_rel(g, gp)


def brute_argmax(d, m):
    """the first strict maximum of each window in row-major order, padding cells excluded: a plain loop"""
    C, H, W = d.shape
    Ho = pgo.pool_out(H, m["kH"], m["dH"], m["padH"], m["ceil_mode"])
    Wo = pgo.pool_out(W, m["kW"], m["dW"], m["padW"], m["ceil_mode"])
    out = np.zeros((C, Ho, Wo), np.int64)
    for c, oy, ox in itertools.product(range(C), range(Ho), range(Wo)):
        best, bi = -np.inf, -1
        for ky, kx in itertools.product(range(m["kH"]), range(m["kW"])):
            y, x = oy * m["dH"] - m["padH"] + ky, ox * m["dW"] - m["padW"] + kx
            if 0 <= y < H and 0 <= x < W and d[c, y, x] > best:
                best, bi = d[c, y, x], y * W + x
        assert bi >= 0
        out[c, oy, ox] = bi
    return out


def pool(kW, kH, dW, dH, padW, padH, ceil):
    return dict(type="pool", kW=kW, kH=kH, dW=dW, dH=dH, padW=padW, padH=padH, ceil_mode=ceil)


POOLS = [pool(2, 2, 2, 2, 0, 0, False), pool(2, 2, 2, 2, 0, 0, True), pool(3, 3, 2, 2, 1, 1, True), pool(3, 3, 1, 1, 1, 1, False),
         pool(2, 2, 1, 1, 0, 0, False), P3x2, pool(3, 2, 2, 1, 1, 0, False), pool(2, 3, 1, 2, 0, 1, True),
         pool(2, 2, 2, 2, 1, 1, True), pool(1, 1, 1, 1, 0, 0, False), pool(4, 1, 3, 1, 2, 0, True)]


@pytest.mark.parametrize("m", POOLS, ids=lambda m: f"k{m['kW']}x{m['kH']}s{m['dW']}x{m['dH']}p{m['padW']}x{m['padH']}"
                                                  f"{'c' if m['ceil_mode'] else 'f'}")
@pytest.mark.parametrize("H,W", [(5, 5), (7, 9), (6, 11), (1, 4)])
def test_argmax_matches_a_loop(m, H, W):
    if H + 2 * m["padH"] < m["kH"] or W + 2 * m["padW"] < m["kW"]:
        pytest.skip("no window fits")
    rng = np.random.default_rng(H * 100 + W)
    d = np.round(rng.standard_normal((4, H, W)) * 2) / 2  # few distinct values: ties everywhere
    d[1] = 0.75                                         # constant windows
    d[2] = -np.abs(d[2]) - 1.0                          # all negative (the padding is not a zero)
    t = torch.from_numpy(d)
    got = pgo.pool_argmax(t, m)
    ref = brute_argmax(d, m)
    assert got.shape == ref.shape and np.array_equal(got.numpy(), ref)
    # the gathered maxima and the extents are F.max_pool2d's
    mp = F.max_pool2d(t[None], (m["kH"], m["kW"]), (m["dH"], m["dW"]), (m["padH"], m["padW"]), ceil_mode=m["ceil_mode"])[0]
    assert torch.equal(pgo.gather(t, got), mp)


def test_argmax_first_of_planted_ties_and_dropped_ceil_window():
    d = torch.zeros(1, 5, 5, dtype=torch.float64)
    d[0, 1, 1] = d[0, 1, 2] = d[0, 2, 1] = 3.0   # one window: three equal maxima, the first in row-major order wins
    m = pool(3, 3, 3, 3, 0, 0, False)
    assert pgo.pool_argmax(d, m)[0, 0, 0] == 1 * 5 + 1
    d[0, 0, 2] = 3.0
    assert pgo.pool_argmax(d, m)[0, 0, 0] == 0 * 5 + 2
    # extent 5, k2 s2 pad 1, ceil: ceil((5 - 2 + 2) / 2) + 1 = 4 windows, but the fourth would start in the padding: 3
    m = pool(2, 2, 2, 2, 1, 1, True)
    assert pgo.pool_out(5, 2, 2, 1, True) == 3 and pgo.pool_argmax(d, m).shape == (1, 3, 3)
    assert F.max_pool2d(d[None], 2, 2, 1, ceil_mode=True).shape[-2:] == (3, 3)


# ---- the per-pixel bar catches what the statistical bar misses ---------------------------------------------------------------

def perturbation_case(name, H, W, seed):
    mods, tested, _, _, agg = chain(name)
    content, stylized, style = images(H, W, seed)
    return mods, tested, agg, net_space(content), net_space(stylized), style


def old_bar_passes(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    d, m = np.abs(got - ref), float(np.abs(ref).max())
    q, l2 = float(np.quantile(d, 0.99)) / m, float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    return q <= OLD_BAR and l2 <= OLD_BAR, (q, l2)


def new_bar_passes(got, ref):
    e, eb = pgo.pixel_err(got, ref)
    return e <= pgo.PIXEL_BAR and eb <= pgo.PIXEL_BAR, (e, eb)


def check_caught(bad, ref, what):
    ok_old, old = old_bar_passes(bad, ref)
    ok_new, new = new_bar_passes(bad, ref)
    print(f"\n{what}: old bar (99%, L2) {old[0]:.1e} {old[1]:.1e}; per-pixel (all, border) {new[0]:.1e} {new[1]:.1e}")
    assert ok_old, (what, old)
    assert not ok_new, (what, new)


def test_style_weight_one_percent_off_is_caught():
    mods, tested, agg, xc, x, style = perturbation_case("pool-k3x2-s2x1-ceil-odd", 20, 31, 5)
    sl, sw = [tested, tested + 1, tested + 2], [0.2, 3.0, 0.2]
    targets = targets_of(mods, sl, sw, agg, style)
    ref, _, _ = pgo.grad(mods, x, xc, [], [], sl, sw, targets, agg)
    assert new_bar_passes(ref, ref)[0]
    bad, _, _ = pgo.grad(mods, x, xc, [], [], sl, [0.2, 3.0 * 1.01, 0.2], targets, agg)
    check_caught(bad, ref, "style weight x 1.01")


def test_zeroed_outer_row_and_column_is_caught():
    """Content loss on a stylized image whose difference from the content image fades towards the borders, so that the
    border carries a small share of the gradient's energy: zeroing the outer row and column moves the L2 error little."""
    mods, tested, agg, xc, _, _ = perturbation_case("cin16-k5", 60, 90, 6)
    yy, xx = np.mgrid[0:60, 0:90]
    taper = torch.from_numpy(np.sin(np.pi * (yy + 0.5) / 60) * np.sin(np.pi * (xx + 0.5) / 90))
    rng = np.random.default_rng(6)
    x = xc + 20.0 * taper ** 2 * torch.from_numpy(rng.standard_normal((3, 60, 90)))
    ref, _, _ = pgo.grad(mods, x, xc, [tested + 1], [1.0], [], [], [], agg)
    bad = ref.clone()
    bad[:, 0, :] = 0
    bad[:, :, 0] = 0
    check_caught(bad, ref, "outer row and column zeroed")


def test_swapped_pooling_window_is_caught():
    """kW and kH swapped in the non-square pooling, as a loss layer next to a heavier one on the raw convolution"""
    mods, tested, agg, xc, x, style = perturbation_case("pool-k3x2-s2x1-ceil-odd", 20, 31, 8)
    sl, sw = [tested, tested + 2], [1.0, 0.002]
    targets = targets_of(mods, sl, sw, agg, style)
    ref, _, _ = pgo.grad(mods, x, xc, [], [], sl, sw, targets, agg)
    swapped = [dict(m) for m in mods]
    swapped[tested + 1].update(kW=P3x2["kH"], kH=P3x2["kW"])
    assert swapped[tested + 1]["type"] == "pool"
    bad, _, _ = pgo.grad(swapped, x, xc, [], [], sl, sw, targets, agg)
    check_caught(bad, ref, "pooling kW / kH swapped")
