"""The single-pass fp16 mode (fav_net_set_precision "fp16", StyleNet.set_precision) on the GPU.
- Per layer, each layer fed the GPU's own input (layer_output of the layer before): against the emulation of the mode
  (tests/fp16_mode_oracle.py: fp16 operands, the packed hi weights, fp64 sums) within fp32 accumulation noise, and against
  the fp64 oracle within a loose bar; the fp64 deviation must be well above the emulator's, which a kernel that still adds the
  lo products, or a mode that never reaches the launch, fails.  IN default arch and every arch-token geometry of
  test_gpu_arch_geometry.py; batch-normalized nets against fp64 (the emulator follows NetOracle's InstanceNorm nets).
- Whole frames (run_image, one run_next_image) at 64x96, 256x256 and 1280x720 within FRAME_BAR of fp64 (about one 8-bit level,
  from the emulator's deviation on the CPU, test_fp16_mode_oracle.py).
- Bit identity within the mode: image b of a batch and the frame alone, the arena plan and the all-live plan, the graph replay
  and the eager first call; switching pair -> fp16 -> pair leaves the exact path bit for bit.
- Surfaces: Session frames, `python -m fav_b200.video -precision fp16`, and a bad mode string refused with FAV_ERR_INVALID.
Clips are not compared across modes: a last-bit change grows to O(1) within tens of recurrent frames (DESIGN.md §2)."""
import glob

import numpy as np
import pytest
import torch

import fp16_mode_oracle as fo
from fav_b200 import _lib, models_video, synth
from test_fp16_mode_oracle import FRAME_BAR
from test_gpu_arch_geometry import BN_ROWS, ROWS
from test_gpu_net import T, rand_input

pytestmark = pytest.mark.gpu

# Per layer.  The emulator's input is layer_output of the layer before, hi + lo of the GPU's operand; the GPU's conv multiplied
# hi = fp16(v).  fp16(hi + lo) differs from hi by one fp16 ulp where v lies within lo's precision of a rounding midpoint (about
# 2^-11 of the elements), so the emulator is off by those flips: on an H100 up to 2.0e-4 max (relative to max(1, max|ref|))
# and 1.3e-5 - 4.4e-5 RMS (relative to the reference's RMS), against 3.8e-4 - 9.8e-4 max and ~4e-4 RMS from fp64.  A kernel
# that still adds the lo products, or a mode that never reaches the launch, sits ~1e-5 from fp64 and ~4e-4 from the emulator.
EMU_MAX_BAR = 5e-4
EMU_RMS_BAR = 1e-4
FP64_BAR = 3e-2    # per layer, max, against the plain fp64 oracle
MARGIN = 4.0       # per conv layer, the RMS deviation from fp64 must exceed the one from the emulator by this factor


def per_layer(net, x, ora_exact, ora_emu):
    """Per layer, each fed the GPU's output of the layer before: dict of lists, max and RMS deviation from the emulator and
    from fp64."""
    net.forward(T(x)[None])
    n = len(ora_exact.specs) - 1
    r = dict(emu_max=[], emu_rms=[], f64_max=[], f64_rms=[])
    inp = torch.from_numpy(x)[None].to(torch.float64)
    for i in range(n):
        g = net.layer_output(i).cpu().numpy().astype(np.float64)
        with torch.no_grad():
            r64 = ora_exact.layer(i, inp)[0].numpy()
            rem = ora_emu.layer(i, inp)[0].numpy()
        s, q = max(1.0, np.abs(r64).max()), max(1e-30, np.sqrt(np.mean(r64 ** 2)))
        r["emu_max"].append(np.abs(g - rem).max() / s)
        r["f64_max"].append(np.abs(g - r64).max() / s)
        r["emu_rms"].append(np.sqrt(np.mean((g - rem) ** 2)) / q)
        r["f64_rms"].append(np.sqrt(np.mean((g - r64) ** 2)) / q)
        inp = torch.from_numpy(g)[None]
    return r


def check_layers(label, net, x, ora_exact, ora_emu):
    r = per_layer(net, x, ora_exact, ora_emu)
    m = {k: max(v) for k, v in r.items()}
    conv = [i for i, sp in enumerate(ora_exact.specs[:len(r["emu_rms"])]) if sp["kind"] != "up"]  # a U token has no conv
    ratio = min(r["f64_rms"][i] / max(r["emu_rms"][i], 1e-30) for i in conv)
    print(f"\n{label}: per layer vs emulator max {m['emu_max']:.2e} rms {m['emu_rms']:.2e}; vs fp64 max {m['f64_max']:.2e} "
          f"rms {m['f64_rms']:.2e}; smallest rms ratio {ratio:.1f}")
    assert m["emu_max"] < EMU_MAX_BAR, (label, r["emu_max"])
    assert m["emu_rms"] < EMU_RMS_BAR, (label, r["emu_rms"])
    assert m["f64_max"] < FP64_BAR, (label, r["f64_max"])
    assert ratio > MARGIN, (label, r["emu_rms"], r["f64_rms"])


def default_pair(style="candy", norm="instance"):
    from oracle import net_oracle
    net = models_video.synthetic_model(style, norm=norm)
    net.set_precision("fp16")
    return net, net_oracle.NetOracle(style=style, dtype=torch.float64), fo.fp16_oracle(style=style)


@pytest.mark.parametrize("shape", [(64, 96), (256, 256)])
def test_default_arch_every_layer(shape):
    net, ex, em = default_pair()
    check_layers(f"default {shape}", net, rand_input(*shape, 5), ex, em)


@pytest.mark.parametrize("name", list(ROWS))
def test_arch_geometry_every_layer(name):
    from oracle import net_oracle
    arch, ptype, in_dim, H, W = ROWS[name]
    w = synth.make_weights(arch, "scream", in_dim)
    net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim, precision="fp16").load_state(w)
    ex = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=in_dim)
    em = fo.fp16_oracle(arch=arch, style="scream", padding_type=ptype, in_dim=in_dim)
    check_layers(name, net, rand_input(H, W, 11)[:in_dim], ex, em)


@pytest.mark.parametrize("name", [None] + BN_ROWS)
def test_batch_norm_every_layer_vs_fp64(name):
    """BN nets (operand epilogue): fp64 within the loose bar, and the single pass measurably off the exact pair path."""
    import bn_oracle
    if name is None:
        arch, ptype, in_dim, H, W = synth.DEFAULT_ARCH, "reflect-start", 7, 64, 96
    else:
        arch, ptype, in_dim, H, W = ROWS[name]
    w = bn_oracle.calibrate_bn_weights(arch, "candy", in_dim, H, W, padding_type=ptype)
    ora = bn_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=w, padding_type=ptype, in_dim=in_dim)
    x = bn_oracle.calibration_input(H, W, in_dim, seed=9)
    dev = {}
    for mode in ("pair", "fp16"):
        net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim, norm="batch", precision=mode).load_state(w)
        taps = {}
        ora.forward(torch.from_numpy(x)[None], taps)
        net.forward(T(x)[None])
        d = 0.0
        for i in range(len(ora.specs) - 1):
            r = taps[f"l{i}"][0].numpy()
            d = max(d, np.abs(net.layer_output(i).cpu().numpy() - r).max() / max(1.0, np.abs(r).max()))
        dev[mode] = d
    print(f"\nBN {name or 'default'}: per layer vs fp64, pair {dev['pair']:.2e}, fp16 {dev['fp16']:.2e}")
    assert dev["fp16"] < FP64_BAR
    assert dev["fp16"] > MARGIN * dev["pair"]


@pytest.mark.parametrize("shape", [(64, 96), (256, 256), (720, 1280)])
def test_whole_frame_vs_fp64(shape):
    from oracle import net_oracle
    H, W = shape
    net = models_video.synthetic_model("candy")
    net.set_precision("fp16")
    ora = net_oracle.NetOracle(style="candy", dtype=torch.float64)
    f1 = synth.make_frame(H, W, 1)
    ref1 = ora.run_image(f1)
    out1 = net.run_image(T(f1)).cpu().numpy()
    e1 = float(np.abs(out1 - ref1).max())
    msg = f"\n{W}x{H}: run_image {e1:.2e}"
    assert e1 < FRAME_BAR, e1
    if H * W <= 256 * 256:
        f2 = synth.make_frame(H, W, 2)
        cert = net_oracle.make_cert(H, W, 2)
        flow = synth.checker_to_lua(synth.make_backward_flow(H, W, 2))
        prev = ref1.astype(np.float32)
        ref2 = ora.run_next_image(f2, prev, flow, cert)
        out2 = net.run_next_image(T(f2), T(prev), T(flow), T(cert)).cpu().numpy()
        e2 = float(np.abs(out2 - ref2).max())
        msg += f", run_next_image {e2:.2e}"
        assert e2 < FRAME_BAR, e2
    print(msg + f" (bar {FRAME_BAR:.1e})")


def test_batch_image_is_the_frame_alone():
    net = models_video.synthetic_model("candy")
    net.set_precision("fp16")
    xs = [rand_input(64, 96, 30 + b) for b in range(3)]
    alone = [net.forward(T(x)[None])[0].cpu() for x in xs]
    out = net.forward(T(np.stack(xs))).cpu()
    for b in range(3):
        assert torch.equal(out[b], alone[b]), b


def test_arena_plan_is_the_all_live_plan():
    live = models_video.synthetic_model("candy")
    arena = models_video.synthetic_model("candy")
    for n in (live, arena):
        n.set_precision("fp16")
    all_live, shared = arena.plan_bytes(64, 96, 2)
    assert shared < all_live
    arena.set_activation_budget(all_live - 1)
    x = T(np.stack([rand_input(64, 96, 40), rand_input(64, 96, 41)]))
    assert torch.equal(live.forward(x), arena.forward(x))


def test_graph_replay_is_the_eager_call():
    net = models_video.synthetic_model("candy")
    net.set_precision("fp16")
    f = T(synth.make_frame(96, 128, 1))
    outs = [net.run_image(f).cpu() for _ in range(4)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_switching_back_restores_the_exact_path():
    a = models_video.synthetic_model("candy")
    b = models_video.synthetic_model("candy")
    f = T(synth.make_frame(64, 96, 1))
    exact = a.run_image(f).clone()
    a.set_precision("fp16")
    single = a.run_image(f).clone()
    a.set_precision("pair")
    again = a.run_image(f)
    assert not torch.equal(single, exact)
    assert torch.equal(again, exact)
    assert torch.equal(b.run_image(f), exact)
    x = T(rand_input(64, 96, 3))[None]
    assert torch.equal(a.forward(x), b.forward(x))


def test_session_frames_are_the_device_api_frames():
    from fav_b200 import consistencyChecker, session, utils
    net = models_video.synthetic_model("candy")
    net.set_precision("fp16")
    H, W = 96, 128
    s = session.Session(net, H, W)
    frames = [torch.from_numpy(synth.make_frame(H, W, i)).pin_memory() for i in range(1, 4)]
    outs = [torch.empty((3, H, W)).pin_memory() for _ in range(3)]
    s.run_image(frames[0], outs[0])
    for i in range(2, 4):
        bw = torch.from_numpy(synth.make_backward_flow(H, W, i)).pin_memory()
        fw = torch.from_numpy(synth.make_forward_flow(H, W, i)).pin_memory()
        s.run_next_image_flows(frames[i - 1], bw, fw, outs[i - 1], 7)
    s.sync()
    prev = net.run_image(frames[0].cuda())
    assert torch.equal(prev.cpu(), outs[0])
    for i in range(2, 4):
        bw, fw = synth.make_backward_flow(H, W, i), synth.make_forward_flow(H, W, i)
        _, cert = consistencyChecker.check(T(bw), T(fw), want_cert=True)
        prev = net.run_next_image(frames[i - 1].cuda(), prev, T(synth.checker_to_lua(bw)), utils.min_filter(cert, 7))
        assert torch.equal(prev.cpu(), outs[i - 1]), i


@pytest.mark.parametrize("pipeline", ["1", "0"])
def test_video_cli_writes_pngs(tmp_path, pipeline):
    from fav_b200 import consistencyChecker, video
    H, W, n = 64, 96, 3
    d = str(tmp_path)
    for i in range(1, n + 1):
        synth.write_ppm(f"{d}/frame_{i:04d}.ppm", synth.make_frame(H, W, i))
    for i in range(2, n + 1):
        synth.write_flo(f"{d}/backward_{i}_{i - 1}.flo", synth.make_backward_flow(H, W, i))
        synth.write_flo(f"{d}/forward_{i - 1}_{i}.flo", synth.make_forward_flow(H, W, i))
        consistencyChecker.main(["consistencyChecker", f"{d}/backward_{i}_{i - 1}.flo", f"{d}/forward_{i - 1}_{i}.flo",
                                 f"{d}/reliable_{i}_{i - 1}.pgm"])
    video.main(["-input_pattern", f"{d}/frame_%04d.ppm", "-flow_pattern", f"{d}/backward_[%d]_{{%d}}.flo",
                "-occlusions_pattern", f"{d}/reliable_[%d]_{{%d}}.pgm", "-output_prefix", f"{d}/out", "-num_frames", str(n),
                "-precision", "fp16", "-pipeline", pipeline])
    assert len(glob.glob(f"{d}/out*.png")) == n


def test_bad_mode_is_refused():
    net = models_video.synthetic_model("candy")
    for bad in ("fp32", "", "FP16", "tf32"):
        with pytest.raises(_lib.FavError) as e:
            net.set_precision(bad)
        assert e.value.status == _lib.FAV_ERR_INVALID
    assert net.precision == "pair"
