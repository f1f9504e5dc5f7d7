"""The loss side of training on the GPU: PerceptualCriterion's forward + backward through the loss network
(fav_percep_forward_backward, csrc/percep.cu), the pixel-loss gradient and the TotalVariation gradient, each against fp64
torch.autograd over the same modules (seeded weights in VGG-16's real shapes)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fav_b200 import _lib, percep, synth
from oracle import percep_oracle

pytestmark = pytest.mark.gpu

# x max |ref|.  Where a pre-activation's fp64 value lies within the forward's rounding of 0 (or a pooling window's two largest
# values do), the ReLU's (pooling's) gradient is discontinuous and either side is right; one such decision deep in the network
# moves the gradient of its whole receptive field, a large share of a 64x96 input.  Measured on an H100: the 99th percentile
# and the relative L2 error stay below 1.2e-2 in every case, the max error below 9e-2; a case without such a unit (the 3x3/2
# pooling one) is 3e-5 off everywhere, and a loss on conv1_1's raw output (no ReLU or pooling on the path) 5e-6.
GRAD_BAR = 2e-2
EXACT_BAR = 1e-3  # max |got - ref| / max |ref| where no ReLU or pooling decision lies on the path
# relative, totals and per-layer losses.  The style loss at relu4_3 is the MSE of (G - T) with G 1.3e-4 off fp64
# (test_gpu_percep.py): 2.3e-4 measured on an H100 at 64x96
LOSS_BAR = 5e-4
STYLE_LAYERS, CONTENT_LAYERS = [4, 9, 16, 23], [16]
MEAN_BGR = torch.tensor(percep_oracle.VGG_MEAN_BGR, dtype=torch.float32)[:, None, None]


def net_space(rgb):
    """preprocess.vgg.preprocess in fp32 (the arithmetic of the evaluate path's fused pack): BGR, x 255, minus the mean"""
    return (torch.from_numpy(np.ascontiguousarray(rgb))[[2, 1, 0]] * 255.0 - MEAN_BGR).contiguous()


def images(H, W, seed):
    rng = np.random.default_rng(seed)
    content = synth.make_frame(H, W, seed)
    stylized = (0.7 * content + 0.3 * rng.uniform(-0.2, 1.2, content.shape)).astype(np.float32)
    yy, xx = np.mgrid[0:70, 0:90]
    style = np.stack([0.5 + 0.5 * np.sin(xx / 3.0 + c) * np.cos(yy / 5.0 - c) for c in range(3)]).astype(np.float32)
    return content, stylized, style


def features(mods, x, indices):
    """percep_oracle.features from a net-space [1,3,H,W] tensor (differentiable)"""
    want, out = set(indices), {}
    for i, m in enumerate(mods[:max(want)], 1):
        if m["type"] == "conv":
            w = torch.as_tensor(np.asarray(m["weight"], np.float64), device=x.device)
            b = torch.as_tensor(np.asarray(m["bias"], np.float64), device=x.device)
            x = F.conv2d(x, w, b, stride=m["stride"], padding=m["pad"])
        elif m["type"] == "relu":
            x = torch.relu(x)
        else:
            x = F.max_pool2d(x, (m["kH"], m["kW"]), (m["dH"], m["dW"]), (m["padH"], m["padW"]), ceil_mode=bool(m["ceil_mode"]))
        if i in want:
            out[i] = x[0]
    return out


def aggregate(f, agg_type):
    C, H, W = f.shape
    x = f.reshape(C, H * W)
    return x @ x.t() / (C * H * W) if agg_type == "gram" else x.mean(1)


def oracle(mods, x, xc, cl, cw, sl, sw, targets, agg_type):
    """fp64 autograd of PerceptualCriterion's output w.r.t. the net-space input: (grad [3,H,W], per-layer losses)"""
    dev = "cuda"
    X = x.to(dev, torch.float64)[None].requires_grad_()
    fc = features(mods, xc.to(dev, torch.float64)[None], cl) if cl else {}
    fs = features(mods, X, cl + sl)
    per = [w * ((fs[i] - fc[i].detach()) ** 2).mean() for i, w in zip(cl, cw)]
    per += [w * ((aggregate(fs[i], agg_type) - t.to(dev)) ** 2).mean() for i, w, t in zip(sl, sw, targets)]
    (g,) = torch.autograd.grad(sum(per), X)
    return g[0].cpu(), [float(v.detach()) for v in per]


def rel_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return float(np.abs(got - ref).max()) / float(np.abs(ref).max())


def grad_err(got, ref):
    """(99th percentile of |got - ref| / max |ref|, relative L2 error, max |got - ref| / max |ref|)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    d, m = np.abs(got - ref), float(np.abs(ref).max())
    return float(np.quantile(d, 0.99)) / m, float(np.linalg.norm(got - ref) / np.linalg.norm(ref)), float(d.max()) / m


def check_grad(got, ref, what):
    q, l2, mx = grad_err(got, ref)
    print(f"  {what}: grad 99% {q:.1e}, L2 {l2:.1e}, max {mx:.1e} of max|ref| {float(np.abs(np.asarray(ref)).max()):.3e}")
    assert q <= GRAD_BAR and l2 <= GRAD_BAR, (what, q, l2, mx)


def setup(mods, cl, cw, sl, sw, agg_type, style):
    crit = percep.PerceptualCriterion(mods, cl, cw, sl, sw, agg_type=agg_type)
    targets = []
    if sl:
        crit.set_style_target(torch.from_numpy(style).cuda())
        targets = percep_oracle.PercepOracle(mods, cl, cw, sl, sw, agg_type).set_style_target(style)
    return crit, targets


def run(crit, x, xc):
    """one fav_percep_forward_backward call -> (grad [3,H,W] cpu, content total, style total, per-layer losses)"""
    import ctypes as C

    xg, cg = x.cuda().contiguous(), xc.cuda().contiguous()
    grad = torch.empty_like(xg)
    n = len(crit.content_layers) + len(crit.style_layers)
    cl, sl, lay = C.c_double(), C.c_double(), (C.c_double * n)()
    _lib.check(_lib.lib.fav_percep_forward_backward(crit._h, _lib.dptr(cg), _lib.dptr(xg), x.shape[1], x.shape[2], _lib.dptr(grad),
                                                    C.byref(cl), C.byref(sl), lay, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return grad.cpu(), cl.value, sl.value, list(lay)


def pool3_modules(seed):
    """VGG-16 with every pooling 3x3 / stride 2 / pad 1 in ceil mode"""
    mods = percep.vgg16_modules(seed)
    for m in mods:
        if m["type"] == "pool":
            m.update(kW=3, kH=3, dW=2, dH=2, padW=1, padH=1, ceil_mode=True)
    return mods


# (name, H, W, modules, content layers, weights, style layers, weights, aggregation)
CASES = [
    ("default mix", 64, 96, lambda: percep.vgg16_modules(11), CONTENT_LAYERS, [1.5], STYLE_LAYERS, [1.0, 2.0, 0.5, 3.0], "gram"),
    ("content on a raw conv", 64, 96, lambda: percep.vgg16_modules(12), [15], [2.0], [], [], "gram"),
    ("content on a pooling", 64, 96, lambda: percep.vgg16_modules(13), [10], [1.0], [], [], "gram"),
    ("style gram on poolings", 64, 96, lambda: percep.vgg16_modules(14), [], [], [5, 10, 17], [1.0, 4.0, 0.25], "gram"),
    ("style mean", 64, 96, lambda: percep.vgg16_modules(15), [], [], STYLE_LAYERS, [1.0, 2.0, 3.0, 4.0], "mean"),
    ("odd extents, ceil", 100, 76, lambda: percep.vgg16_modules(16, ceil_mode=True), [17], [1.0], [16, 23], [2.0, 1.0], "gram"),
    ("odd extents, floor", 100, 76, lambda: percep.vgg16_modules(17), [23], [1.0], [18, 19], [1.0, 1.0], "gram"),
    ("3x3/2 pad 1 ceil pooling", 66, 90, lambda: pool3_modules(18), [10], [1.0], [5, 16], [1.0, 2.0], "gram"),
    ("content and style on conv1_1", 64, 96, lambda: percep.vgg16_modules(19), [1], [1.0], [1], [2.0], "gram"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_grad_and_losses_vs_fp64_autograd(case):
    name, H, W, make, cl, cw, sl, sw, agg_type = case
    mods = make()
    content, stylized, style = images(H, W, 3)
    crit, targets = setup(mods, cl, cw, sl, sw, agg_type, style)
    x, xc = net_space(stylized), net_space(content)
    grad, tc, ts, lay = run(crit, x, xc)
    ref, per = oracle(mods, x, xc, cl, cw, sl, sw, targets, agg_type)
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    print(f"\n{name} {H}x{W}: layers " + " ".join(f"{v:.1e}" for v in lay_e))
    check_grad(grad, ref, name)
    if max(cl + sl) == 1:
        assert grad_err(grad, ref)[2] <= EXACT_BAR
    assert max(lay_e) <= LOSS_BAR, (name, lay_e)
    rc, rs = sum(per[:len(cl)]), sum(per[len(cl):])
    assert (not cl or abs(tc - rc) <= LOSS_BAR * abs(rc)) and (not sl or abs(ts - rs) <= LOSS_BAR * abs(rs)), (tc, rc, ts, rs)


def test_losses_match_evaluate_and_repeat_bitwise():
    mods = percep.vgg16_modules(21)
    content, stylized, style = images(64, 96, 4)
    sw = [1.0, 2.0, 0.5, 3.0]
    crit, _ = setup(mods, CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, "gram", style)
    ec, es = crit.evaluate(torch.from_numpy(content).cuda(), torch.from_numpy(stylized).cuda())
    x, xc = net_space(stylized), net_space(content)
    g1, c1, s1, l1 = run(crit, x, xc)
    assert abs(c1 - ec) <= 1e-6 * abs(ec) and abs(s1 - es) <= 1e-6 * abs(es), (c1, ec, s1, es)
    assert abs(sum(l1[1:]) - s1) <= 1e-12 * s1 and l1[0] == c1
    # the evaluate path keeps its own plan and results after a backward call
    assert crit.evaluate(torch.from_numpy(content).cuda(), torch.from_numpy(stylized).cuda()) == (ec, es)
    g2, c2, s2, l2 = run(crit, x, xc)
    assert torch.equal(g1, g2) and (c1, s1, l1) == (c2, s2, l2)


def test_tiny_gradient_keeps_the_bar():
    """A content weight that puts max |grad| near 1e-11: the per-tensor power-of-two scale keeps the fp16 operands normal."""
    mods = percep.vgg16_modules(22)
    content, stylized, style = images(64, 96, 6)
    x, xc = net_space(stylized), net_space(content)
    ref1, _ = oracle(mods, x, xc, [9, 16], [1.0, 1.0], [], [], [], "gram")
    w = 1e-11 / float(ref1.abs().max())
    crit, _ = setup(mods, [9, 16], [w, w], [], [], "gram", style)
    grad, tc, _, _ = run(crit, x, xc)
    ref, per = oracle(mods, x, xc, [9, 16], [w, w], [], [], [], "gram")
    assert float(ref.abs().max()) < 1e-10
    check_grad(grad, ref, "tiny")
    assert abs(tc - sum(per)) <= LOSS_BAR * sum(per)
    # identical input and target: a zero gradient everywhere, zeros and not NaN
    grad0, tc0, _, _ = run(crit, xc, xc)
    assert tc0 == 0.0 and torch.equal(grad0, torch.zeros_like(grad0))


def test_stride2_conv_before_the_loss_layer_is_refused():
    mods = percep.vgg16_modules(23)[:9]
    mods[5] = dict(mods[5], stride=2)  # conv2_1 (module 6) at stride 2, pad 1
    content, stylized, _ = images(64, 96, 7)
    crit = percep.PerceptualCriterion(mods, [9], [1.0], [], [])
    assert crit.evaluate(torch.from_numpy(content).cuda(), torch.from_numpy(stylized).cuda())[0] > 0  # the forward still runs
    with pytest.raises(_lib.FavError) as e:
        run(crit, net_space(stylized), net_space(content))
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "module 6" in str(e.value)


def test_batch_through_the_python_api():
    mods = percep.vgg16_modules(24)
    H, W = 64, 96
    c1, s1, style = images(H, W, 8)
    c2, s2, _ = images(H, W, 9)
    sw = [1.0, 2.0, 0.5, 3.0]
    crit, targets = setup(mods, CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, "gram", style)
    x = torch.stack([net_space(s1), net_space(s2)]).cuda()
    xc = torch.stack([net_space(c1), net_space(c2)]).cuda()
    target = {"content_target": xc}
    total = crit.forward(x, target)
    grad = crit.backward(x, target)
    assert grad.shape == (2, 3, H, W)
    refs = [oracle(mods, x[n].cpu(), xc[n].cpu(), CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, targets, "gram") for n in range(2)]
    per = [(a + b) / 2 for a, b in zip(refs[0][1], refs[1][1])]
    for n in range(2):
        check_grad(grad[n].cpu(), refs[n][0] / 2, f"image {n}")
    assert abs(total - sum(per)) <= LOSS_BAR * sum(per)
    assert len(crit.content_losses) == 1 and len(crit.style_losses) == 4
    for got, ref in zip(crit.content_losses + crit.style_losses, per):
        assert abs(got - ref) <= LOSS_BAR * ref
    assert abs(crit.total_content_loss + crit.total_style_loss - total) <= 1e-12 * total


@pytest.mark.parametrize("loss_type", ["L2", "L1", "SmoothL1"])
def test_pixel_loss_grad_vs_fp64_autograd(loss_type):
    rng = np.random.default_rng(30)
    N, H, W, weight = 2, 37, 53, 0.7
    out2 = torch.from_numpy((rng.standard_normal((N, 3, H, W)) * 2).astype(np.float32))
    prev = torch.from_numpy((rng.standard_normal((N, 3, H, W)) * 2).astype(np.float32))
    cert = torch.from_numpy(rng.uniform(0, 1, (N, 1, H, W)).astype(np.float32))  # not binary: the gradient is NOT multiplied by it
    acc0 = torch.from_numpy((rng.standard_normal((N, 3, H, W)) * 1e-5).astype(np.float32))  # fp32 ulps stay below the bar
    acc = acc0.cuda()
    loss = percep.pixel_loss_grad(out2.cuda(), prev.cuda(), cert.cuda(), loss_type, weight, acc)
    a = (out2.double() * cert.double()).requires_grad_()
    crit = {"L2": torch.nn.MSELoss(), "L1": torch.nn.L1Loss(), "SmoothL1": torch.nn.SmoothL1Loss()}[loss_type]
    ref = weight * crit(a, prev.double())
    (g,) = torch.autograd.grad(ref, a)
    got = acc.cpu().double() - acc0.double()
    assert abs(loss - float(ref)) <= 1e-6 * float(ref), (loss, float(ref))
    assert rel_err(got, g) <= 1e-5, rel_err(got, g)


def test_tv_grad_vs_fp64_autograd():
    rng = np.random.default_rng(31)
    N, H, W, strength = 2, 29, 41, 1e-3
    x = torch.from_numpy((rng.standard_normal((N, 3, H, W)) * 50).astype(np.float32))
    acc0 = torch.from_numpy((rng.standard_normal((N, 3, H, W)) * 0.01).astype(np.float32))
    acc = acc0.cuda()
    percep.tv_grad(x.cuda(), strength, acc)
    X = x.double().requires_grad_()
    xd = X[:, :, :-1, :-1] - X[:, :, :-1, 1:]
    yd = X[:, :, :-1, :-1] - X[:, :, 1:, :-1]
    (g,) = torch.autograd.grad(strength * 0.5 * ((xd ** 2).sum() + (yd ** 2).sum()), X)
    assert rel_err(acc.cpu().double() - acc0.double(), g) <= 1e-5


def test_grad_at_1280x720_vs_fp64_autograd():
    mods = percep.vgg16_modules(25)
    H, W = 720, 1280
    content, stylized, style = images(H, W, 10)
    sw = [1.0, 2.0, 0.5, 3.0]
    crit, targets = setup(mods, CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, "gram", style)
    x, xc = net_space(stylized), net_space(content)
    grad, tc, ts, lay = run(crit, x, xc)
    ref, per = oracle(mods, x, xc, CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, targets, "gram")
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    print("\n1280x720: layers " + " ".join(f"{v:.1e}" for v in lay_e))
    check_grad(grad, ref, "1280x720")
    assert max(lay_e) <= LOSS_BAR, lay_e
