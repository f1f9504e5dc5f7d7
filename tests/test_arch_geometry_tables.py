"""The arch table of test_gpu_arch_geometry.py on the CPU: it reaches every geometry an arch token can give the stylization
net's planner, every arch in it gets past planning in fav_net_finalize, and the token geometries the planner cannot run are
refused there, by layer name, before any device work.  Also pins why the frame size must be checked against the arch: the
oracle returns a larger frame than it was given when a stride-2 layer sees an odd size."""
import pytest
import torch

from fav_b200 import synth
from test_gpu_arch_geometry import BATCH_ROW, BN_ROWS, ROWS, THREE_S2
from test_wide_tables import _finalize_error


def geometries(arch, in_dim):
    """(position, Cin, k, stride) of each conv, ('full', k, stride) of each transposed conv, ('U', scale) of each nearest
    upsampling, ('block', scale) of each residual / conv block (scale: input pixels per pixel)"""
    specs = synth.parse_arch(arch, in_dim)
    out, scale = set(), 1
    for i, s in enumerate(specs):
        if s["kind"] == "conv":
            out.add(("first" if i == 0 else "final" if i == len(specs) - 1 else "conv", s["cin"], s["k"], s["stride"]))
            scale *= s["stride"]
        elif s["kind"] == "fullconv":
            out.add(("full", s["k"], s["stride"]))
            scale //= s["stride"]
        elif s["kind"] == "up":
            out.add(("U", s["scale"]))
            scale //= s["scale"]
        else:
            out.add(("block", scale))
    return out


REQUIRED = (
    {("first", cin, k, 1) for cin in (7, 3) for k in (1, 3, 5, 7)}                 # tap pairing
    | {("conv", 64, 1, 1), ("conv", 128, 1, 1), ("conv", 32, 5, 1), ("conv", 64, 5, 1), ("conv", 64, 7, 1), ("conv", 16, 9, 1)}
    | {("final", 32, 7, 1), ("final", 16, 7, 1), ("final", 32, 1, 1), ("final", 8, 5, 1)}  # x-fold k 7, generic, tap pairing
    | {("full", k, 1) for k in (1, 5, 7, 9)} | {("full", 7, 2), ("full", 9, 2)}
    | {("U", 1), ("U", 4)}
)


def test_gpu_table_covers_every_arch_token_geometry():
    """Trimming the table must not silently drop a geometry."""
    geo = {name: geometries(arch, in_dim) for name, (arch, _, in_dim, _, _) in ROWS.items()}
    found = set().union(*geo.values())
    assert REQUIRED <= found, sorted(REQUIRED - found)
    # residual / conv blocks at two scales, in both padding types
    mixed = {ROWS[n][1] for n, g in geo.items() if len({t for t in g if t[0] == "block"}) >= 2}
    assert mixed == {"reflect-start", "zero"}
    # three stride-2 layers at a size they restore
    assert any(sum(s["kind"] == "conv" and s["stride"] == 2 for s in synth.parse_arch(a, d)) == 3 and H % 8 == 0 and W % 8 == 0
               for a, _, d, H, W in ROWS.values())
    # x-fold frame widths at the tile edges: k 5 strides 124 pixels, k 7 strides 122
    edges = {(k, W) for n, (a, _, d, _, W) in ROWS.items() for (pos, cin, k, _) in
             (t for t in geo[n] if t[0] == "final") if cin >= 16 and k >= 5}
    assert {(5, 248), (5, 252), (7, 244), (7, 248)} <= edges, sorted(edges)
    # batch-normalized rows: operand epilogues into consumers with padT 3 / 4 and tpad 2 - 4
    bn = set().union(*(geo[n] for n in BN_ROWS))
    assert {("conv", 64, 7, 1), ("conv", 16, 9, 1), ("full", 5, 1), ("full", 7, 1), ("full", 9, 1)} <= bn
    assert any(t[0] == "full" and t[2] == 2 for t in geo[BATCH_ROW])


@pytest.mark.parametrize("name,norm", [(n, "instance") for n in ROWS] + [(n, "batch") for n in BN_ROWS])
def test_gpu_table_archs_pass_planning(name, norm):
    """Every arch of the GPU table plans: finalize gets past the planner (without a GPU it then stops at the device)."""
    from fav_b200 import _lib

    arch, ptype, in_dim, _, _ = ROWS[name]
    e = _finalize_error(arch, ptype, in_dim, norm)
    if torch.cuda.is_available():
        assert e is None, e
    else:
        assert e is not None and e.status == _lib.FAV_ERR_NO_DEVICE, e


@pytest.mark.parametrize("arch,layer", [
    ("c9s1-32,c5s2-64,d128,R128,u64,u32,c9s1-3", "l1"),        # stride 2 runs k 3 pad 1 only
    ("c9s1-32,c7s2-64,d128,R128,u64,u32,c9s1-3", "l1"),
    ("c9s1-32,c9s2-64,d128,R128,u64,u32,c9s1-3", "l1"),
    ("c3s2-32,d64,R64,u32,u16,c9s1-3", "l0"),                  # stride 2 from 7 channels: the parity split needs Cin % 16 == 0
    ("c9s1-32,d64,R64,u128,c5s1-3", "l4"),                     # x-fold from 128: 5 filter rows, a prime, need 20 K groups
    ("c9s1-32,d64,R64,u128,c7s1-3", "l4"),                     # ... 7 rows need 28 (9 rows split in 3: the table's U4 row)
    ("c9s1-32,d64,d128,c5s1-128,R128,u64,u32,c9s1-3", "l3"),   # non-final 5x5 / 7x7 from 128: more than 16 K groups
    ("c9s1-32,d64,d128,c7s1-128,R128,u64,u32,c9s1-3", "l3"),
    ("c9s1-32,d64,d128,u32,f1s2-16,c9s1-3", "l4"),             # f1s2: sub-pixel phases without filter taps (from 32 ...
    ("c9s1-32,d64,d128,u8,f1s2-16,c9s1-3", "l4"),              # ... and from 8 channels, tap pairing)
])
def test_unplannable_token_geometries_are_refused_at_finalize(arch, layer):
    from fav_b200 import _lib

    e = _finalize_error(arch)
    assert e is not None and e.status == _lib.FAV_ERR_UNSUPPORTED, e
    assert f"conv {layer}:" in str(e), str(e)
    if "f1s2" in arch:
        assert "without filter taps" in str(e), str(e)


@pytest.mark.parametrize("shape,out", [((68, 68), (72, 72)), ((72, 100), (72, 104)), ((72, 104), (72, 104))])
def test_oracle_frame_size_of_three_stride2_layers(shape, out):
    """With three stride-2 layers 68 + 32 (reflection pad) = 100 -> 50 -> 25 -> 13 -> 9 (residual block) -> 18 -> 36 -> 72:
    the net returns a larger frame than it was given, so the final conv's [3][H][W] output cannot hold it and fav_net_* refuse
    the size.  Multiples of 8 are restored."""
    from oracle import net_oracle

    ora = net_oracle.NetOracle(arch=THREE_S2, style="scream", dtype=torch.float32)
    y = ora.forward(torch.zeros((1, 7) + shape))
    assert tuple(y.shape) == (1, 3) + out
