"""The activation arena on the GPU.  A plan whose buffers exceed the net's activation budget (fav_net_set_activation_budget)
puts its operands in one arena by lifetime (arena_plan.hpp) and zeroes each operand's border right before the step that
writes it.  The kernels and their order are those of the all-live plan, so with the budget one byte below the all-live total
every output is bit-identical to the all-live plan's.  The arena starts out filled with fp16 NaNs, so a border a consumer
reads without its clear would show up as a difference.  Layers whose activation a later layer took over are refused by
fav_net_layer_output; the input of the final layer stays readable.  One 7680x4320 frame runs at the default budget."""
import gc

import pytest
import torch

from fav_b200 import _lib, models_video, synth

pytestmark = pytest.mark.gpu

WIDE = "c9s1-32,d64,d256,C256,f3s1-192,u96,u32,c9s1-3"


def frames(B, H, W, n, seed):
    """n frames of B clips: content, backward flow (dy, dx) and forward flow (u, v) of a few pixels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lead = (B,) if B > 1 else ()
    out = []
    for _ in range(n):
        img = torch.rand(lead + (3, H, W), generator=g, device="cuda")
        bw = torch.randn(lead + (2, H, W), generator=g, device="cuda") * 3
        fw = torch.randn(lead + (2, H, W), generator=g, device="cuda") * 3
        out.append((img, bw, fw))
    return out


def pair(arch=synth.DEFAULT_ARCH, norm="instance", B=1, H=64, W=96):
    """The same net twice: all-live plan (default budget), and an arena plan (budget one byte below the all-live total)."""
    live = models_video.synthetic_model("candy", arch, norm=norm)
    arena = models_video.synthetic_model("candy", arch, norm=norm)
    all_live, shared = arena.plan_bytes(H, W, B)
    assert shared < all_live
    arena.set_activation_budget(all_live - 1)
    return live, arena, all_live, shared


def run_clip(net, clip):
    """run_image on the first frame, then run_next_image_flows (occlusions from the flow pair) on each further frame."""
    img, _, _ = clip[0]
    outs = [net.run_image(img)]
    for img, bw, fw in clip[1:]:
        outs.append(net.run_next_image_flows(img, outs[-1], bw, fw, None, 7))
    torch.cuda.synchronize()
    return outs


def free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("shape", [(64, 96), (720, 1280), (2160, 3840)], ids=["64x96", "720p", "4K"])
def test_arena_bit_identical_recurrence(shape):
    H, W = shape
    live, arena, all_live, shared = pair(H=H, W=W)
    clip = frames(1, H, W, 6, seed=H)
    a, b = run_clip(live, clip), run_clip(arena, clip)
    print(f"{W}x{H}: all-live {all_live / 2**30:.2f} GiB, arena plan {shared / 2**30:.2f} GiB")
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.isfinite(x).all()
        assert torch.equal(x, y), f"frame {i}: max diff {(x - y).abs().max().item()}"
    del live, arena, clip, a, b
    free()


@pytest.mark.parametrize("arch,norm", [(synth.DEFAULT_ARCH, "instance"), (synth.DEFAULT_ARCH, "batch"), (WIDE, "instance")],
                         ids=["IN", "BN", "wide"])
def test_arena_bit_identical_batch_1080p(arch, norm):
    B, H, W = 2, 1080, 1920
    live, arena, _, _ = pair(arch, norm, B, H, W)
    clip = frames(B, H, W, 3, seed=7)
    a, b = run_clip(live, clip), run_clip(arena, clip)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.isfinite(x).all()
        assert torch.equal(x, y), f"frame {i}: max diff {(x - y).abs().max().item()}"
    x = torch.rand((B, 7, H, W), device="cuda") * 100
    assert torch.equal(live.forward(x), arena.forward(x))
    del live, arena, clip, a, b
    free()


@pytest.mark.parametrize("arch,norm", [(synth.DEFAULT_ARCH, "instance"), (synth.DEFAULT_ARCH, "batch"),
                                       (synth.PAPER_ARCH, "instance")], ids=["IN", "BN", "paper"])
def test_arena_layer_outputs(arch, norm):
    """Taken-over layers raise FAV_ERR_INVALID naming the layer; the others, the final layer's input among them, read back
    the all-live plan's bits."""
    H, W = 64, 96
    live, arena, _, _ = pair(arch, norm, 1, H, W)
    x = torch.rand((1, 7, H, W), device="cuda") * 100
    assert torch.equal(live.forward(x), arena.forward(x))
    n = len(arch.split(",")) - 1
    refused = []
    for i in range(n):
        try:
            got = arena.layer_output(i)
        except _lib.FavError as e:
            assert e.status == _lib.FAV_ERR_INVALID and f"layer {i} " in e.message, e.message
            refused.append(i)
            continue
        assert torch.equal(got, live.layer_output(i)), f"layer {i}"
    assert refused and n - 1 not in refused, refused


def test_budget_refusal_names_both_figures():
    net = models_video.synthetic_model("candy")
    all_live, shared = net.plan_bytes(64, 96)
    net.set_activation_budget(shared // 2)
    with pytest.raises(_lib.FavError) as e:
        net.run_image(torch.rand((3, 64, 96), device="cuda"))
    assert e.value.status == _lib.FAV_ERR_INVALID
    assert "shared between layers" in e.value.message and "budget" in e.value.message, e.value.message


def test_8k_frame_default_budget():
    H, W = 4320, 7680
    net = models_video.synthetic_model("candy")
    all_live, shared = net.plan_bytes(H, W)
    assert all_live > 32 << 30 >= shared, (all_live, shared)
    img = torch.rand((3, H, W), device="cuda")
    out1 = torch.empty_like(img)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    _lib.check(_lib.lib.fav_run_image(net._h, _lib.dptr(img), None, H, W, _lib.dptr(out1), _lib.stream_ptr()))
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    took = free0 - free1
    print(f"8K plan: planner {shared / 2**30:.2f} GiB shared ({all_live / 2**30:.2f} GiB all-live), device memory taken "
          f"{took / 2**30:.2f} GiB")
    assert shared <= took <= shared + (1 << 30), (shared, took)
    out2 = net.run_image(img)
    torch.cuda.synchronize()
    assert torch.isfinite(out1).all()
    assert torch.equal(out1, out2)
    del net, img, out1, out2
    free()
