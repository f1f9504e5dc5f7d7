"""Batches on the GPU: B frames of one size through one plan, every kernel covering all B images in one launch (conv.cuh
tile_at).  Image b of a batch must be bit-identical to the same image run alone -- at every layer tap, at the output and
through run_image / run_next_image / run_next_image_flows and the lockstep clip driver -- and within the fp64 oracle's bars of
test_gpu_net.py: 2e-4 * max|ref| per layer, TOL / 10 on the deprocessed frame."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from fav_b200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3
WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rand_input(H, W, seed, in_dim=7):
    from oracle import pyoracle

    rng = np.random.default_rng(seed)
    x7 = pyoracle.first_frame_input(synth.make_frame(H, W, 1 + seed % 5))
    x7[3:6] = rng.normal(0, 50, (3, H, W))
    x7[6] = rng.uniform(0, 1, (H, W))
    return x7[:in_dim].astype(np.float32)


@functools.lru_cache(maxsize=None)
def bn_weights(arch):
    import bn_oracle

    return bn_oracle.calibrate_bn_weights(arch, "candy", 7, 64, 96)


def make_case(arch, ptype, in_dim, norm):
    from fav_b200 import models_video
    from oracle import net_oracle

    if norm == "batch":
        import bn_oracle

        w = bn_weights(arch)
        net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim, norm="batch").load_state(w)
        ora = bn_oracle.NetOracle(arch=arch, dtype=torch.float64, weights=w, padding_type=ptype, in_dim=in_dim)
        return net, ora
    w = synth.make_weights(arch, "scream", in_dim)
    net = models_video.StyleNet(arch, padding_type=ptype, in_dim=in_dim).load_state(w)
    ora = net_oracle.NetOracle(arch=arch, style="scream", dtype=torch.float64, padding_type=ptype, in_dim=in_dim)
    return net, ora


def taps_of(net, n_layers, b=0):
    return [net.layer_output(i, b).cpu() for i in range(n_layers)]


# 48x508: output widths of the residual convs cross 128-pixel tile edges
@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
@pytest.mark.parametrize("arch,ptype,in_dim,norm", [
    (synth.DEFAULT_ARCH, "reflect-start", 7, "instance"),
    (synth.DEFAULT_ARCH, "zero", 7, "instance"),
    (synth.PAPER_ARCH, "reflect-start", 7, "instance"),
    (synth.DEFAULT_ARCH, "reflect-start", 7, "batch"),
    (WIDE, "reflect-start", 7, "instance"),
    (synth.DEFAULT_ARCH, "reflect-start", 3, "instance"),
])
def test_batched_forward_is_each_image_alone_and_matches_oracle(arch, ptype, in_dim, norm, shape):
    H, W = shape
    B = 3
    net, ora = make_case(arch, ptype, in_dim, norm)
    if norm == "batch":
        import bn_oracle

        xs = [bn_oracle.calibration_input(H, W, seed=9 + b) for b in range(B)]
    else:
        xs = [rand_input(H, W, 9 + b, in_dim) for b in range(B)]
    n_layers = len(ora.specs) - 1
    alone, alone_taps = [], []
    for x in xs:
        alone.append(net.forward(T(x)[None]).cpu()[0])
        alone_taps.append(taps_of(net, n_layers))
    out = net.forward(T(np.stack(xs))).cpu()
    assert out.shape == (B, 3, H, W)
    for b, x in enumerate(xs):
        assert torch.equal(out[b], alone[b]), f"image {b}: batched output differs from the image run alone"
        batched_taps = taps_of(net, n_layers, b)
        taps = {}
        ref = ora.forward(torch.from_numpy(x)[None], taps)[0].numpy()
        for i in range(n_layers):
            assert torch.equal(batched_taps[i], alone_taps[b][i]), f"image {b}, layer {i}: not bit-identical"
            r = taps[f"l{i}"][0].numpy()
            g = batched_taps[i].numpy()
            assert np.abs(g - r).max() < 2e-4 * max(1.0, np.abs(r).max()), f"image {b}, layer {i}"
        assert np.abs(out[b].numpy() - ref).max() / 255.0 < TOL / 10


@pytest.fixture(scope="module")
def default_net():
    from fav_b200 import models_video

    return models_video.synthetic_model("candy")


def clip_inputs(H, W, B, seed=0):
    from oracle import net_oracle

    frames = np.stack([synth.make_frame(H, W, 2 + b) for b in range(B)])
    prev = np.stack([synth.make_frame(H, W, 7 + b) for b in range(B)])
    flows = np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 2 + b)) for b in range(B)])
    fws = np.stack([synth.make_forward_flow(H, W, 2 + b) for b in range(B)])
    certs = np.stack([net_oracle.make_cert(H, W, 2 + b) for b in range(B)])
    return T(frames), T(prev), T(flows), T(fws), T(certs)


@pytest.mark.parametrize("shape", [(64, 96), (48, 508)])
def test_batched_frame_calls_are_per_image_calls(default_net, shape):
    H, W = shape
    B = 3
    frames, prev, flows, fws, certs = clip_inputs(H, W, B)
    net = default_net
    got = net.run_image(frames)
    for b in range(B):
        assert torch.equal(got[b], net.run_image(frames[b])), f"run_image, image {b}"
    got = net.run_next_image(frames, prev, flows, certs)
    for b in range(B):
        assert torch.equal(got[b], net.run_next_image(frames[b], prev[b], flows[b], certs[b])), f"run_next_image, image {b}"
    # the whole temporal stage with the occlusion test on the GPU and the min filter
    got = net.run_next_image_flows(frames, prev, flows, fws, None, 7)
    for b in range(B):
        one = net.run_next_image_flows(frames[b], prev[b], flows[b], fws[b], None, 7)
        assert torch.equal(got[b], one), f"run_next_image_flows, image {b}"
    got = net.run_next_image_flows(frames, prev, flows, None, certs, 7)
    for b in range(B):
        assert torch.equal(got[b], net.run_next_image_flows(frames[b], prev[b], flows[b], None, certs[b], 7))


def test_lockstep_clips_equal_single_clip_runs(default_net):
    from fav_b200 import clips
    from oracle import net_oracle

    H, W, B, n = 64, 96, 3, 3
    frames = T(np.stack([np.stack([synth.make_frame(H, W, 1 + 3 * c + i) for i in range(n)]) for c in range(B)]))
    flows = T(np.stack([np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 1 + c + i)) for i in range(n)])
                        for c in range(B)]))
    certs = T(np.stack([np.stack([net_oracle.make_cert(H, W, 1 + c + i) for i in range(n)]) for c in range(B)]))
    got = clips.run_clips_lockstep(default_net, frames, flows, certs)
    for c in range(B):
        one = clips.run_clips_lockstep(default_net, frames[c:c + 1], flows[c:c + 1], certs[c:c + 1])[0]
        prev = None
        for i in range(n):  # the plain single-frame calls
            ref = default_net.run_image(frames[c, i]) if i == 0 else \
                default_net.run_next_image(frames[c, i], prev, flows[c, i], certs[c, i])
            assert torch.equal(got[c, i], ref) and torch.equal(one[i], ref), f"clip {c}, frame {i}"
            prev = ref


@pytest.mark.parametrize("shape,B", [
    ((720, 1280), 2),
    ((256, 256), 2),  # residual convs: 64..82 tiles per image (one wave), 128..164 for the batch (two waves)
])
def test_batched_large_and_wave_crossing(default_net, shape, B):
    H, W = shape
    xs = [rand_input(H, W, 3 + b) for b in range(B)]
    out = default_net.forward(T(np.stack(xs))).cpu()
    for b, x in enumerate(xs):
        assert torch.equal(out[b], default_net.forward(T(x)[None]).cpu()[0]), f"image {b}"


def test_alternating_batch_sizes_keep_single_frame_outputs(default_net):
    """Plans and CUDA graphs are cached per (B, H, W) and destination: interleaving batched calls must not disturb them."""
    H, W = 64, 96
    frames, prev, flows, _, certs = clip_inputs(H, W, 2)
    out1 = torch.empty_like(frames[0])
    refs = []
    for k in range(3):
        r = default_net.run_next_image(frames[0], prev[0], flows[0], certs[0])
        refs.append(r)
        out1.copy_(default_net.run_image(frames[0]))
        got2 = default_net.run_next_image(frames, prev, flows, certs)
        assert torch.equal(got2[0], refs[0])
    a = default_net.run_image(frames[0])
    assert torch.equal(a, out1)
    assert all(torch.equal(r, refs[0]) for r in refs)


@pytest.mark.parametrize("norm", ["instance", "batch"])
def test_batch_agrees_with_cuda_core_comparator(norm):
    arch = synth.DEFAULT_ARCH
    net, _ = make_case(arch, "reflect-start", 7, norm)
    H, W, B = 64, 96, 3
    x = T(np.stack([rand_input(H, W, 20 + b) for b in range(B)]))
    tc = net.forward(x).cpu()
    net.set_conv_impl("simt")
    try:
        simt = net.forward(x).cpu()
    finally:
        net.set_conv_impl("tcgen05")
    for b in range(B):
        assert torch.equal(simt[b], net_simt_single(net, x[b]))
        assert (tc[b] - simt[b]).abs().max().item() / 255.0 < TOL / 10, f"image {b}"


def net_simt_single(net, x1):
    net.set_conv_impl("simt")
    try:
        return net.forward(x1[None]).cpu()[0]
    finally:
        net.set_conv_impl("tcgen05")


def test_invalid_batches_are_refused(default_net):
    from fav_b200 import _lib

    H, W = 64, 96
    net = default_net
    x = torch.zeros((1, 7, H, W), device="cuda")
    out = torch.empty((1, 3, H, W), device="cuda")
    for B in (0, -1, 65):
        rc = _lib.lib.fav_net_forward_batch(net._h, _lib.dptr(x), B, H, W, _lib.dptr(out), None)
        assert rc == _lib.FAV_ERR_INVALID, (B, rc)
        rc = _lib.lib.fav_run_image_batch(net._h, _lib.dptr(x), None, B, H, W, _lib.dptr(out), None)
        assert rc == _lib.FAV_ERR_INVALID, (B, rc)
    # activations of 64 1920x1080 frames do not fit the per-plan cap: refused before anything is allocated or launched
    rc = _lib.lib.fav_run_image_batch(net._h, _lib.dptr(x), None, 64, 1080, 1920, _lib.dptr(out), None)
    assert rc == _lib.FAV_ERR_INVALID and "batch" in _lib.last_error()
    with pytest.raises(_lib.FavError) as e:
        net.layer_output(0, 5)
    assert e.value.status == _lib.FAV_ERR_INVALID
    frames, prev, flows, fws, certs = clip_inputs(H, W, 2)
    for bad in (dict(prev_rgb=prev[:1]), dict(flow=flows[..., :-1]), dict(cert=certs[:, None, None])):
        kw = dict(prev_rgb=prev, flow=flows, cert=certs)
        kw.update(bad)
        with pytest.raises(_lib.FavError) as e:
            net.run_next_image(frames, **kw)
        assert e.value.status == _lib.FAV_ERR_INVALID
    with pytest.raises(_lib.FavError):
        net.run_next_image_flows(frames, prev, flows, fws[:1], None, 7)
    with pytest.raises(_lib.FavError):
        net.run_image(frames, fill=torch.zeros((3, H, W), device="cuda"))
    assert torch.equal(net.run_image(frames)[1], net.run_image(frames[1]))  # still usable afterwards
