"""The stylization net at the sizes the activation arena opened: 7680x4320 frames and a batch of nine 3840x2160 frames.

  * 8K, every layer against fp64 (default arch, InstanceNorm; the all-live plan, so every layer can be read).  Each layer is
    computed by the oracle in fp64 on the GPU (cuDNN) from the product's own previous layer (teacher forced), so each layer's
    error stands alone; then the oracle runs free from the same input.  The oracle's input is the C oracle's consistency ->
    min_filter(7) -> temporal_input, the composition the fused temporal stage equals bit for bit, so layer 0 also checks the
    fused front end at 8K.  1280x720 runs the same checks as the control.  The fused InstanceNorm statistics keep fp32 partial
    sums per CTA over all of its tiles of an image (55 tiles at 720p, 1,964 at 8K), so the error of each IN layer is printed
    with the largest |mean|/std of its input channels.
  * 8K arena plan == all-live plan, bit for bit, over run_image and two recurrent frames (IN at the default budget; BN, whose
    all-live plan fits the default budget, one byte below its all-live total).
  * A batch of nine 4K frames: the first layer's tensor spans more than 2^31 elements, so every batch offset has to be 64-bit;
    each image equals, bit for bit, the same image run alone.
  * fav_temporal_stage at 8K == the C oracle composition, bit for bit.

Each case runs the product and then the oracle, never both at once; the largest is the 34.6 GiB all-live 8K plan.  A case
skips, with the figures, when the device or the host has too little free memory for it."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from fav_b200 import _lib, models_video, synth

pytestmark = pytest.mark.gpu

GiB = 1 << 30
H8K, W8K = 4320, 7680
ALL_LIVE_BUDGET = 40 * GiB  # above the 34.58 GiB all-live 8K plan
DEFAULT_BUDGET = 32 * GiB   # fav_net_set_activation_budget's default
# max|got - ref| <= LAYER_BAR * max(1, max|ref|) per layer, teacher forced.  Measured on an H100 80GB HBM3 (700 W): the worst
# layer uses 0.26 of its bar at 720p and 0.33 at 8K (DESIGN.md §8).
LAYER_BAR = 2e-5
FRAME_BAR = 1e-4            # deprocessed frame, free running (the 4K bar of test_gpu_parity_large.py)


def free():
    gc.collect()
    torch.cuda.empty_cache()


def host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def need_device(nbytes, what):
    torch.cuda.synchronize()
    avail, total = torch.cuda.mem_get_info()
    if avail < nbytes:
        pytest.skip(f"{what}: needs {nbytes / GiB:.1f} GiB of device memory, {avail / GiB:.1f} GiB free of {total / GiB:.1f} GiB")


def need_host(nbytes, what):
    avail = host_available()
    if avail < nbytes:
        pytest.skip(f"{what}: needs {nbytes / GiB:.1f} GiB of host memory, {avail / GiB:.1f} GiB available")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def layer_shape(net, i):
    c, h, w = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib.fav_net_layer_output_image(net._h, i, 0, None, C.byref(c), C.byref(h), C.byref(w), None))
    return c.value, h.value, w.value


def max_abs_diff(got, ref):
    """max |got - ref| of a host fp32 CxHxW tensor and a device 1xCxHxW one, one channel at a time (an 8K layer in fp64 is
    8.7 GB; its difference is not materialized whole)."""
    return max((got[c].cuda().double() - ref[0, c]).abs().max().item() for c in range(got.size(0)))


# ---- 1. every layer against fp64 at 720p and 8K ------------------------------------------------------------------------
def temporal_case(H, W):
    """Frame 2 of the synthetic clip with an unclamped prior in [-0.1, 1.1] and a flow pair of a few pixels; x7 is the C
    oracle's net input for it."""
    from oracle import pyoracle

    frame = synth.make_frame(H, W, 2)
    prev = (synth.make_frame(H, W, 1) * 1.2 - 0.1).astype(np.float32)
    bw, fw = synth.make_backward_flow(H, W, 2), synth.make_forward_flow(H, W, 2)
    flow = synth.checker_to_lua(bw)
    cert = pyoracle.min_filter(pyoracle.consistency(bw, fw).astype(np.float32) / 255.0, 7)
    x7 = pyoracle.temporal_input(frame, prev, flow, cert)
    return frame, prev, flow, fw, x7


def run_product(H, W, inputs):
    """One run_next_image_flows frame on the all-live plan -> (output, every layer's activation), on the host."""
    frame, prev, flow, fw, _ = inputs
    net = models_video.synthetic_model("candy")
    net.set_activation_budget(ALL_LIVE_BUDGET)
    all_live, _ = net.plan_bytes(H, W)
    assert all_live <= ALL_LIVE_BUDGET, all_live
    need_device(all_live + 56 * H * W + 4 * 32 * (H + 80) * (W + 80) + GiB, f"{W}x{H} all-live plan ({all_live / GiB:.2f} GiB)")
    out = net.run_next_image_flows(T(frame), T(prev), T(flow), T(fw), None, 7).cpu()
    n = len(synth.parse_arch(synth.DEFAULT_ARCH)) - 1
    host = sum(4 * np.prod(layer_shape(net, i)) for i in range(n))
    need_host(host + 2 * GiB, f"{W}x{H}: every layer on the host")
    layers = [net.layer_output(i).cpu() for i in range(n)]
    del net
    free()
    return out, layers


def check_against_fp64(H, W):
    """-> (rows, failures): per layer (name, kind, err, bar, max|ref|, IN input |mean|/std or None)."""
    from oracle import net_oracle

    inputs = temporal_case(H, W)
    out, layers = run_product(H, W, inputs)
    x7 = torch.from_numpy(inputs[4])[None]
    ora = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    n = len(ora.specs)
    biggest = max(4 * l.numel() for l in layers)
    need_device(4 * 2 * biggest + GiB, f"{W}x{H} fp64 oracle")
    ora.to("cuda")
    rows, failures = [], []

    def ratio_hook(ratios):
        def hook(name, t):
            var, mean = torch.var_mean(t, dim=(2, 3), unbiased=False)
            ratios.append((mean.abs() / var.sqrt()).max().item())
        return hook

    for i in range(n):
        s = ora.specs[i]
        ratios = []
        x = (x7 if i == 0 else layers[i - 1]).cuda()
        with torch.no_grad():
            ref = ora.layer(i, x if i == 0 else x[None], ratio_hook(ratios))
        del x
        if i < n - 1:
            assert tuple(layers[i].shape) == tuple(ref.shape[1:]), (i, layers[i].shape, ref.shape)
            err, mref = max_abs_diff(layers[i], ref), ref.abs().max().item()
            name = f"l{i}"
        else:  # the final layer through tanh and deprocess, against the frame the product returned
            ref = ora.deprocess(torch.tanh(ref) * ora.tanh_constant)
            err, mref = max_abs_diff(out, ref), ref.abs().max().item()
            name = f"l{i} (deprocessed)"
        bar = LAYER_BAR * max(1.0, mref)
        rows.append((name, s["kind"], err, bar, mref, max(ratios) if ratios else None))
        if not err <= bar:
            failures.append(f"{W}x{H} layer {name}: max|got - ref| {err:.3e} > {bar:.3e} (max|ref| {mref:.3f})")
        del ref
        free()
    with torch.no_grad():
        ref = ora.deprocess(ora.forward(x7.cuda()))
    err = max_abs_diff(out, ref)
    rows.append(("frame (free-running oracle)", "", err, FRAME_BAR, ref.abs().max().item(), None))
    if not err <= FRAME_BAR:
        failures.append(f"{W}x{H} frame vs free-running fp64 oracle: {err:.3e} > {FRAME_BAR:.1e}")
    del ora, ref, layers, out
    free()
    return rows, failures


def test_every_layer_vs_fp64_720p_and_8k():
    results, failures = {}, []
    for H, W in ((720, 1280), (H8K, W8K)):
        rows, fails = check_against_fp64(H, W)
        results[(H, W)] = rows
        failures += fails
    for (H, W), rows in results.items():
        print(f"\n{W}x{H}, default arch, InstanceNorm: teacher-forced layers and the free-running frame vs fp64")
        for name, kind, err, bar, mref, ratio in rows:
            r = "" if ratio is None else f"  IN input max |mean|/std {ratio:.2f}"
            print(f"  {name:<28} {kind:<8} err {err:.2e}  bar {bar:.2e}  max|ref| {mref:8.3f}{r}")
    assert not failures, "\n".join(failures)


# ---- 2. the 8K arena plan equals the all-live plan ----------------------------------------------------------------------
def clip_8k(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(3):
        img = torch.rand((3, H8K, W8K), generator=g, device="cuda")
        bw = torch.randn((2, H8K, W8K), generator=g, device="cuda") * 3
        fw = torch.randn((2, H8K, W8K), generator=g, device="cuda") * 3
        out.append((img, bw, fw))
    return out


def run_clip(net, clip):
    """run_image on the first frame, then run_next_image_flows on each further one -> outputs on the host."""
    outs = [net.run_image(clip[0][0])]
    for img, bw, fw in clip[1:]:
        outs.append(net.run_next_image_flows(img, outs[-1], bw, fw, None, 7))
    torch.cuda.synchronize()
    return [o.cpu() for o in outs]


@pytest.mark.parametrize("norm", ["instance", "batch"], ids=["IN", "BN"])
def test_8k_arena_equals_all_live(norm):
    net = models_video.synthetic_model("candy", norm=norm)
    all_live, shared = net.plan_bytes(H8K, W8K)
    arena_budget = DEFAULT_BUDGET if all_live > DEFAULT_BUDGET else all_live - 1
    assert shared <= arena_budget < all_live <= ALL_LIVE_BUDGET, (all_live, shared)
    need_device(all_live + 3 * 28 * H8K * W8K + GiB, f"8K all-live plan ({all_live / GiB:.2f} GiB)")
    clip = clip_8k(seed=8)
    net.set_activation_budget(ALL_LIVE_BUDGET)
    live = run_clip(net, clip)
    del net
    free()
    net = models_video.synthetic_model("candy", norm=norm)
    net.set_activation_budget(arena_budget)
    arena = run_clip(net, clip)
    print(f"\n8K {norm}: all-live {all_live / GiB:.2f} GiB, arena plan {shared / GiB:.2f} GiB (budget {arena_budget / GiB:.2f} GiB)")
    del net, clip
    free()
    bad = [f"frame {i}: max diff {(x - y).abs().max().item()}" for i, (x, y) in enumerate(zip(live, arena)) if not torch.equal(x, y)]
    assert all(torch.isfinite(x).all() for x in live)
    assert not bad, f"8K {norm}: arena plan differs from the all-live plan: " + "; ".join(bad)


# ---- 3. nine 4K frames in one batch: tensors past 2^31 elements ---------------------------------------------------------
def test_batch_of_nine_4k_frames_equals_each_image_alone():
    B, H, W = 9, 2160, 3840
    specs = synth.parse_arch(synth.DEFAULT_ARCH)
    pad = synth.reflect_start_pad(specs)
    first = B * specs[0]["cout"] * (H + 2 * pad) * (W + 2 * pad)
    assert first > 2**31 - 1, first  # the first layer's fp32 tensor: offsets past it need 64 bits
    net = models_video.synthetic_model("candy")
    net.set_activation_budget(ALL_LIVE_BUDGET)
    all_live, shared = net.plan_bytes(H, W, B)
    assert shared <= ALL_LIVE_BUDGET < all_live, (all_live, shared)  # the arena plan
    need_device(shared + B * 48 * H * W + GiB, f"nine 4K frames (arena plan {shared / GiB:.2f} GiB)")
    g = torch.Generator(device="cuda").manual_seed(9)
    img1 = torch.rand((B, 3, H, W), generator=g, device="cuda")
    img2 = torch.rand((B, 3, H, W), generator=g, device="cuda")
    bw = torch.randn((B, 2, H, W), generator=g, device="cuda") * 3
    fw = torch.randn((B, 2, H, W), generator=g, device="cuda") * 3
    out1 = net.run_image(img1)
    out2 = net.run_next_image_flows(img2, out1, bw, fw, None, 7)
    torch.cuda.synchronize()
    print(f"\nnine 4K frames: first layer {first / 2**31:.2f} x 2^31 elements; all-live {all_live / GiB:.2f} GiB, "
          f"arena plan {shared / GiB:.2f} GiB")
    del net
    free()
    one = models_video.synthetic_model("candy")
    bad = []
    for b in range(B):
        a1 = one.run_image(img1[b])
        a2 = one.run_next_image_flows(img2[b], out1[b], bw[b], fw[b], None, 7)
        for k, (x, y) in enumerate(((out1[b], a1), (out2[b], a2))):
            if not torch.equal(x, y):
                bad.append(f"image {b} frame {k}: max diff {(x - y).abs().max().item()}")
    assert torch.isfinite(out1).all() and torch.isfinite(out2).all()
    assert not bad, "batch of nine 4K frames differs from each image alone: " + "; ".join(bad)
    del one, img1, img2, bw, fw, out1, out2
    free()


# ---- 4. the fused temporal stage at 8K ----------------------------------------------------------------------------------
def test_temporal_stage_8k_bit_exact():
    """fav_temporal_stage (occlusion test or given certainty -> min filter -> warp -> preprocess -> mask -> concat) at 8K,
    both border modes, == the C oracle composition, as test_gpu_front.py checks it at 360x640."""
    from oracle import pyoracle

    H, W = H8K, W8K
    need_device(40 * H * W + GiB, "8K temporal stage")
    c, p = synth.make_frame(H, W, 2), synth.make_frame(H, W, 1) * 1.2 - 0.1
    bw, fw = synth.make_backward_flow(H, W, 2), synth.make_forward_flow(H, W, 2)
    flow = synth.checker_to_lua(bw)
    rng = np.random.default_rng(12)
    fill = rng.normal(0, 40, size=(3, H, W)).astype(np.float32)
    fmask = rng.uniform(size=(H, W)).astype(np.float32)
    cert_given = (rng.uniform(size=(H, W)) > 0.15).astype(np.float32)
    computed = pyoracle.min_filter(pyoracle.consistency(bw, fw).astype(np.float32) / 255.0, 7)
    tc, tp, tflow, tfw = T(c), T(p), T(flow), T(fw)
    out = torch.empty((7, H, W), device="cuda")
    cert_out = torch.empty((H, W), device="cuda")
    bad = []
    for border in (0, 1):
        for given, f, m in ((None, None, None), (cert_given, fill, fmask)):
            tgiven, tfill, tm = (T(a) if a is not None else None for a in (given, f, m))
            _lib.check(_lib.lib.fav_temporal_stage(_lib.dptr(tc), _lib.dptr(tp), _lib.dptr(tflow),
                                                   None if given is not None else _lib.dptr(tfw), _lib.dptr(tgiven),
                                                   _lib.dptr(tfill), _lib.dptr(tm), _lib.dptr(out), _lib.dptr(cert_out), H, W,
                                                   7, border, _lib.stream_ptr()))
            ocert = computed if given is None else pyoracle.min_filter(given, 7)
            ref = pyoracle.temporal_input(c, p, flow, ocert, f, m, warp_mode=border)
            got, gcert = out.cpu().numpy(), cert_out.cpu().numpy()
            what = f"border {border}, {'computed' if given is None else 'given'} certainty"
            if not np.array_equal(gcert, ocert):
                bad.append(f"{what}: certainty differs at {int((gcert != ocert).sum())} pixels")
            if not np.array_equal(got, ref):
                bad.append(f"{what}: net input differs at {int((got != ref).sum())} values, max diff {np.abs(got - ref).max()}")
    assert not bad, "; ".join(bad)
