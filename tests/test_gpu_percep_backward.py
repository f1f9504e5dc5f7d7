"""The loss side of training on the GPU: PerceptualCriterion's forward + backward through the loss network
(fav_percep_forward_backward, csrc/percep.cu), the pixel-loss gradient and the TotalVariation gradient, each against fp64
torch.autograd over the same modules: VGG-16's real shapes with seeded weights, and every geometry of the loss-network sweep
(test_gpu_conv_geometry.CASES).  The loss network's gradient is checked at every pixel against an fp64 chain that takes the
GPU's ReLU and pooling decisions (oracle/percep_grad_oracle.py)."""
import numpy as np
import pytest
import torch

from fav_b200 import _lib, percep, synth
from oracle import percep_grad_oracle as pgo
from oracle import percep_oracle
from test_gpu_conv_geometry import CASES as GEOMETRY, backward_refusal, chain, conv
from test_gpu_percep import FEATURE_BAR, cuda

pytestmark = pytest.mark.gpu

# The reference gradient (oracle/percep_grad_oracle.py) takes the ReLU masks and pooling arg-maxes the backward pass read from
# its fp32 conv outputs (fav_percep_conv_output), so it is a linear map of continuous values and is compared at every pixel:
# max |got - ref| <= PIXEL_BAR x max |ref|, over the whole gradient and over its outer two rows and columns on their own.
# Every unit where a GPU decision differs from the fp64 forward's own must lie within the forward's feature bar of the
# discontinuity: |z| (or the window's fp64 gap to its maximum) <= FEATURE_BAR x max |z| of its conv output.
PIXEL_BAR = pgo.PIXEL_BAR
EXACT_BAR = 1e-3  # max |got - ref| / max |ref| against plain fp64 autograd, where no ReLU or pooling decision lies on the path
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


def rel_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return float(np.abs(got - ref).max()) / float(np.abs(ref).max())


def check_backward(crit, mods, grad, x, xc, cl, cw, sl, sw, targets, agg_type, what, scale=1.0):
    """The checks of one fav_percep_forward_backward result `grad` (x scale = the reference's factor) against the fixed-decision
    fp64 reference; the conv outputs are those of the last call.  Returns (reference gradient, per-layer losses)."""
    last = max(list(cl) + list(sl))
    convs = [i for i, m in enumerate(mods[:last], 1) if m["type"] == "conv"]
    raws = {i: crit.conv_output(i) for i in convs}
    with torch.no_grad():
        f64 = pgo.plain_features(mods, x.to("cuda", torch.float64), convs)
    feat = max(rel_err(raws[i].cpu(), f64[i].cpu()) for i in convs)
    del f64
    ref, per, dec = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, agg_type, raws=raws, device="cuda")
    ref = ref * scale
    e, eb = pgo.pixel_err(grad, ref)
    l2 = float(np.linalg.norm(np.asarray(grad, np.float64) - ref.numpy()) / np.linalg.norm(ref.numpy()))
    ndiff, worst = sum(d[2] for d in dec), max([d[3] for d in dec], default=0.0)
    print(f"  {what}: grad max {e:.1e}, border {eb:.1e}, L2 {l2:.1e} of max|ref| {float(ref.abs().max()):.3e}; conv outputs "
          f"{feat:.1e}; {ndiff} decisions differ from fp64 (worst {worst:.1e})")
    assert feat <= FEATURE_BAR, (what, feat)
    assert e <= PIXEL_BAR and eb <= PIXEL_BAR, (what, e, eb)
    assert worst <= FEATURE_BAR, (what, [d for d in dec if d[2]])
    return ref, per


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
    print(f"\n{name} {H}x{W}:")
    ref, per = check_backward(crit, mods, grad, x, xc, cl, cw, sl, sw, targets, agg_type, name)
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    print("  layers " + " ".join(f"{v:.1e}" for v in lay_e))
    if max(cl + sl) == 1:
        plain, _, _ = pgo.grad(mods, x, xc, cl, cw, sl, sw, targets, agg_type, device="cuda", plain=True)
        assert rel_err(grad, plain) <= EXACT_BAR
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
    ref1, _, _ = pgo.grad(mods, x, xc, [9, 16], [1.0, 1.0], [], [], [], "gram", device="cuda", plain=True)
    w = 1e-11 / float(ref1.abs().max())
    crit, _ = setup(mods, [9, 16], [w, w], [], [], "gram", style)
    grad, tc, _, _ = run(crit, x, xc)
    print()
    ref, per = check_backward(crit, mods, grad, x, xc, [9, 16], [w, w], [], [], [], "gram", "tiny")
    assert float(ref.abs().max()) < 1e-10
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
    print()
    refs = []
    for n in range(2):
        # the same image alone: bitwise the batch's gradient x N, and its conv outputs are the ones the batch decided from
        gn, _, _, _ = run(crit, x[n].cpu(), xc[n].cpu())
        assert torch.equal(gn * 0.5, grad[n].cpu())
        refs.append(check_backward(crit, mods, grad[n].cpu(), x[n].cpu(), xc[n].cpu(), CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw,
                                   targets, "gram", f"image {n}", scale=0.5))
    per = [(a + b) / 2 for a, b in zip(refs[0][1], refs[1][1])]
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
    print()
    ref, per = check_backward(crit, mods, grad, x, xc, CONTENT_LAYERS, [1.5], STYLE_LAYERS, sw, targets, "gram", "1280x720")
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    print("  layers " + " ".join(f"{v:.1e}" for v in lay_e))
    assert max(lay_e) <= LOSS_BAR, lay_e


def geometry_layers(mods, tested):
    """the loss layers of test_gpu_conv_geometry: the tested conv's raw output and every module after it, content on the
    first and the last"""
    layers = list(range(tested, len(mods) + 1))
    return [tested, layers[-1]], [1.0, 0.5], layers, [1.0 + 0.5 * i for i in range(len(layers))]


def check_refused(crit, x, xc, content, stylized, module):
    n0 = _lib.lib.fav_launch_count()
    with pytest.raises(_lib.FavError) as e:
        run(crit, x, xc)
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and f"module {module}:" in str(e.value), str(e.value)
    assert _lib.lib.fav_launch_count() == n0
    with pytest.raises(_lib.FavError) as e2:
        crit.conv_output(1)  # no backward plan ran since the style target
    assert e2.value.status == _lib.FAV_ERR_INVALID
    cl, sl = crit.evaluate(cuda(content), cuda(stylized))
    assert cl > 0 and sl > 0


@pytest.mark.parametrize("name", list(GEOMETRY))
def test_backward_over_the_geometry_table(name):
    """Every loss-network geometry of the forward sweep either backpropagates under the per-pixel checks or is refused by
    the rules (test_gpu_conv_geometry.backward_refusal) before any kernel runs, leaving evaluate working."""
    mods, tested, H, W, agg = chain(name)
    cl, cw, sl, sw = geometry_layers(mods, tested)
    content, stylized, style = images(H, W, 7)
    crit, targets = setup(mods, cl, cw, sl, sw, agg, style)
    x, xc = net_space(stylized), net_space(content)
    refusal = backward_refusal(mods)
    print(f"\n{name} {H}x{W}: " + (f"refused at module {refusal[0]} ({refusal[1]})" if refusal else ""))
    if refusal:
        check_refused(crit, x, xc, content, stylized, refusal[0])
        return
    grad, tc, ts, lay = run(crit, x, xc)
    _, per = check_backward(crit, mods, grad, x, xc, cl, cw, sl, sw, targets, agg, name)
    lay_e = [abs(a - b) / abs(b) for a, b in zip(lay, per)]
    assert max(lay_e) <= LOSS_BAR, lay_e
    # the evaluate plans share one raw buffer: the hook answers for backward plans only
    crit.evaluate(cuda(content), cuda(stylized))
    with pytest.raises(_lib.FavError) as e:
        crit.conv_output(tested)
    assert e.value.status == _lib.FAV_ERR_INVALID
    crit.close()


def stage_terms_modules(n_relu, relu_after_pool):
    rng = np.random.default_rng(40 + n_relu)
    R = dict(type="relu")
    mods = [conv(rng, 3, 16, 3, 1, 1)] + [dict(R) for _ in range(n_relu)] + [dict(type="pool", kW=2, kH=2, dW=2, dH=2, padW=0,
                                                                                   padH=0, ceil_mode=False)]
    mods += [dict(R)] * relu_after_pool + [conv(rng, 16, 32, 3, 1, 1), dict(R)]
    return mods


def test_seven_loss_layers_on_one_stage_and_an_eighth_refused():
    """conv1's stage carries the raw conv, five ReLUs and the pooling as loss layers (content and style mixed) next to the
    term of the next stage: the eight terms percep_bwd_stage_kernel takes.  One more loss layer there is refused."""
    content, stylized, style = images(20, 36, 12)
    x, xc = net_space(stylized), net_space(content)
    mods = stage_terms_modules(5, 0)
    cl, cw, sl, sw = [1, 4, 7, 9], [1.0, 0.5, 2.0, 0.3], [2, 3, 5, 6, 7, 9], [1.0, 1.5, 0.5, 2.0, 1.0, 0.7]
    crit, targets = setup(mods, cl, cw, sl, sw, "gram", style)
    grad, tc, ts, lay = run(crit, x, xc)
    print()
    _, per = check_backward(crit, mods, grad, x, xc, cl, cw, sl, sw, targets, "gram", "seven layers on stage 1")
    assert max(abs(a - b) / abs(b) for a, b in zip(lay, per)) <= LOSS_BAR
    mods = stage_terms_modules(5, 1)  # conv, five ReLUs, pooling, ReLU: eight loss layers before the next conv
    crit, _ = setup(mods, [1, 4, 8, 10], cw, sl, sw, "gram", style)
    check_refused(crit, x, xc, content, stylized, 1)
