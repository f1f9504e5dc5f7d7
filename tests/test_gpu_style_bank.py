"""Style banks on the GPU (fav_net_add_style, fav_net_set_batch_styles): one net holding several weight sets of its architecture,
each image of a batch with its own style.  Image b must be bit-identical to the same input run alone on the net its style came
from -- through run_image, a recurrent run_next_image_flows clip, every layer tap, the CUDA-core comparator, an arena plan and
the lockstep clip driver -- and a bank without an assignment must give the bits its own net gave."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from fav_b200 import _lib, synth

pytestmark = pytest.mark.gpu

PAPER = synth.PAPER_ARCH
DOUBLED = "c9s1-64,d128,d256,R256,R256,u128,u64,c9s1-3"
STYLES = ("candy", "mosaic", "udnie")
ASSIGN = [2, 0, 1, 2]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def weights(arch, style, norm, in_dim=7):
    if norm == "batch":
        import bn_oracle

        return bn_oracle.calibrate_bn_weights(arch, style, in_dim, 64, 96)
    return synth.make_weights(arch, style, in_dim)


def style_net(arch, style, ptype="reflect-start", norm="instance", precision="pair", in_dim=7, tanh_constant=150.0):
    from fav_b200 import models_video

    return models_video.StyleNet(arch, ptype, tanh_constant=tanh_constant, in_dim=in_dim, norm=norm,
                                 precision=precision).load_state(weights(arch, style, norm, in_dim))


def make_bank(arch, ptype="reflect-start", norm="instance", precision="pair"):
    """(bank, nets): the bank holds STYLES[s] as style s; nets[s] is that style's own net."""
    nets = [style_net(arch, s, ptype, norm, precision) for s in STYLES]
    bank = style_net(arch, STYLES[0], ptype, norm, precision)
    for s in range(1, len(STYLES)):
        assert bank.add_style(style_net(arch, STYLES[s], ptype, norm, precision)) == s
    assert bank.num_styles == len(STYLES)
    return bank, nets


def clip(H, W, B, n):
    """n frames of B clips: frames [n,B,3,H,W], backward flows (dy,dx) and forward flows (u,v) [n,B,2,H,W]."""
    frames = T(np.stack([np.stack([synth.make_frame(H, W, 1 + 3 * b + i) for b in range(B)]) for i in range(n)]))
    flows = T(np.stack([np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 1 + b + i)) for b in range(B)])
                        for i in range(n)]))
    fws = T(np.stack([np.stack([synth.make_forward_flow(H, W, 1 + b + i) for b in range(B)]) for i in range(n)]))
    return frames, flows, fws


def check_against_style_nets(bank, nets, assign, H, W, n=3):
    frames, flows, fws = clip(H, W, len(assign), n)
    got = bank.run_image(frames[0], styles=assign)
    refs = [nets[s].run_image(frames[0, b]) for b, s in enumerate(assign)]
    for b in range(len(assign)):
        assert torch.equal(got[b], refs[b]), f"run_image, image {b} (style {assign[b]})"
    prev = got
    for i in range(1, n):
        got = bank.run_next_image_flows(frames[i], prev, flows[i], fws[i], None, 7, styles=assign)
        refs = [nets[s].run_next_image_flows(frames[i, b], refs[b], flows[i, b], fws[i, b], None, 7) for b, s in enumerate(assign)]
        for b in range(len(assign)):
            assert torch.equal(got[b], refs[b]), f"run_next_image_flows frame {i}, image {b} (style {assign[b]})"
        prev = got


@pytest.mark.parametrize("shape", [(64, 96), (256, 256), (720, 1280)])
@pytest.mark.parametrize("arch,ptype,norm,precision", [
    (synth.DEFAULT_ARCH, "reflect-start", "instance", "pair"),
    (synth.DEFAULT_ARCH, "reflect-start", "instance", "fp16"),
    (PAPER, "reflect-start", "instance", "pair"),
    (DOUBLED, "reflect-start", "instance", "pair"),
    (synth.DEFAULT_ARCH, "zero", "instance", "pair"),
    (synth.DEFAULT_ARCH, "reflect-start", "batch", "pair"),
])
def test_each_image_equals_its_style_net(arch, ptype, norm, precision, shape):
    bank, nets = make_bank(arch, ptype, norm, precision)
    check_against_style_nets(bank, nets, ASSIGN, *shape)


def test_arena_plan_with_styles():
    """Two 1920x1080 frames under a budget below the all-live plan: the operands share an arena, each image runs its style."""
    bank, nets = make_bank(synth.DEFAULT_ARCH)
    H, W = 1080, 1920
    all_live, shared = bank.plan_bytes(H, W, 2)
    assert shared < all_live
    bank.set_activation_budget((shared + all_live) // 2)
    check_against_style_nets(bank, nets, [1, 2], H, W, n=2)


def test_every_layer_of_each_image_is_its_style_nets():
    bank, nets = make_bank(synth.DEFAULT_ARCH)
    H, W = 64, 96
    from oracle import pyoracle

    xs = [pyoracle.first_frame_input(synth.make_frame(H, W, 1 + b)).astype(np.float32) for b in range(len(ASSIGN))]
    bank.forward(T(np.stack(xs)), styles=ASSIGN)
    n_layers = len(synth.DEFAULT_ARCH.split(",")) - 1
    got = [[bank.layer_output(i, b).cpu() for i in range(n_layers)] for b in range(len(ASSIGN))]
    for b, s in enumerate(ASSIGN):
        nets[s].forward(T(xs[b][None]))
        for i in range(n_layers):
            assert torch.equal(got[b][i], nets[s].layer_output(i).cpu()), f"layer {i}, image {b} (style {s})"


@pytest.mark.parametrize("norm", ["instance", "batch"])
def test_cuda_core_comparator_mixed_batch(norm):
    bank, nets = make_bank(synth.DEFAULT_ARCH, norm=norm)
    H, W = 64, 96
    from oracle import pyoracle

    xs = T(np.stack([pyoracle.first_frame_input(synth.make_frame(H, W, 2 + b)).astype(np.float32) for b in range(len(ASSIGN))]))
    bank.set_conv_impl("simt")
    got = bank.forward(xs, styles=ASSIGN)
    for b, s in enumerate(ASSIGN):
        nets[s].set_conv_impl("simt")
        assert torch.equal(got[b], nets[s].forward(xs[b:b + 1])[0]), f"image {b} (style {s})"


def test_defaults_and_switching_assignments():
    from fav_b200 import models_video

    H, W = 256, 256
    frames, _, _ = clip(H, W, 4, 1)
    net = style_net(synth.DEFAULT_ARCH, STYLES[0])
    before = net.run_image(frames[0])
    one = [net.run_image(frames[0, b]) for b in range(4)]
    net.add_style(style_net(synth.DEFAULT_ARCH, STYLES[1]))
    # no assignment: every image runs style 0, the net's own weights, with the bits it gave before add_style
    assert torch.equal(net.run_image(frames[0]), before)
    assert torch.equal(net.run_image(frames[0, 1]), one[1])
    # every image on style 1 = a plain batch on style 1's net
    ref1 = style_net(synth.DEFAULT_ARCH, STYLES[1]).run_image(frames[0])
    assert torch.equal(net.run_image(frames[0], styles=[1, 1, 1, 1]), ref1)
    # A -> B -> A on one plan (and its graph) gives A's bits again
    a = net.run_image(frames[0], styles=[0, 1, 0, 1])
    b = net.run_image(frames[0], styles=[1, 0, 1, 0])
    assert torch.equal(net.run_image(frames[0], styles=[0, 1, 0, 1]), a)
    assert torch.equal(b[0], ref1[0]) and torch.equal(b[1], before[1])
    assert isinstance(net, models_video.StyleNet)


def test_refusals_and_source_lifetime():
    from fav_b200 import models_video

    arch = synth.DEFAULT_ARCH
    bank = style_net(arch, STYLES[0])

    def refused(other, what):
        idx = C.c_int(-1)
        assert _lib.lib.fav_net_add_style(bank._h, other._h, C.byref(idx)) == _lib.FAV_ERR_INVALID, what
        assert what in _lib.last_error(), (what, _lib.last_error())

    refused(style_net(PAPER, STYLES[1]), "arch")
    refused(style_net(arch, STYLES[1], ptype="zero"), "padding_type")
    refused(style_net(arch, STYLES[1], norm="batch"), "norm")
    refused(style_net(arch, STYLES[1], in_dim=3), "in_dim")
    refused(style_net(arch, STYLES[1], tanh_constant=100.0), "tanh_constant")
    refused(models_video.StyleNet(arch), "finalized")
    assert bank.num_styles == 1
    # a style outlives the net it was copied from
    src = style_net(arch, STYLES[1])
    assert bank.add_style(src) == 1
    del src
    H, W = 64, 96
    frames, _, _ = clip(H, W, 2, 1)
    assert torch.equal(bank.run_image(frames[0], styles=[1, 0])[0], style_net(arch, STYLES[1]).run_image(frames[0, 0]))
    with pytest.raises(_lib.FavError) as e:
        bank.run_image(frames[0], styles=[0, 2])  # index out of range
    assert e.value.status == _lib.FAV_ERR_INVALID
    with pytest.raises(_lib.FavError) as e:
        bank.run_image(frames[0], styles=[0, 1, 1])  # B != n
    assert e.value.status == _lib.FAV_ERR_INVALID
    # at most 64 styles
    tiny = "c9s1-16,c9s1-3"
    small = models_video.StyleNet(tiny).load_state(synth.make_weights(tiny, STYLES[0]))
    other = models_video.StyleNet(tiny).load_state(synth.make_weights(tiny, STYLES[1]))
    for _ in range(63):
        small.add_style(other)
    assert small.num_styles == 64
    with pytest.raises(_lib.FavError) as e:
        small.add_style(other)
    assert e.value.status == _lib.FAV_ERR_INVALID and "64" in e.value.message


def test_lockstep_clips_in_their_styles():
    from fav_b200 import clips
    from oracle import net_oracle

    bank, nets = make_bank(synth.DEFAULT_ARCH)
    H, W, n = 64, 96, 3
    assign = [1, 2, 0]
    B = len(assign)
    frames = T(np.stack([np.stack([synth.make_frame(H, W, 1 + 3 * c + i) for i in range(n)]) for c in range(B)]))
    flows = T(np.stack([np.stack([synth.checker_to_lua(synth.make_backward_flow(H, W, 1 + c + i)) for i in range(n)])
                        for c in range(B)]))
    certs = T(np.stack([np.stack([net_oracle.make_cert(H, W, 1 + c + i) for i in range(n)]) for c in range(B)]))
    got = clips.run_clips_lockstep(bank, frames, flows, certs, styles=assign)
    for c, s in enumerate(assign):
        one = clips.run_clips_lockstep(nets[s], frames[c:c + 1], flows[c:c + 1], certs[c:c + 1])[0]
        assert torch.equal(got[c], one), f"clip {c} (style {s})"
