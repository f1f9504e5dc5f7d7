"""The oracle of the single-pass fp16 mode (tests/fp16_mode_oracle.py) on the CPU:
- without rounding, its hook reproduces NetOracle exactly;
- its weights are the hi halves the product packs (fp16(w 2^e) 2^-e) and differ from the weights by at most 2^-11 relative;
- its whole-frame deviation from the fp64 oracle at 256x256 (seeded default arch) is the expected error of the mode, about one
  8-bit level of the deprocessed frame: the bar the GPU tests (test_gpu_fp16_mode.py) use, FRAME_BAR."""
import numpy as np
import torch

import fp16_mode_oracle as fo
from fav_b200 import synth

# whole-frame max-abs of the mode against fp64 on the deprocessed [0,1] frame: the emulator's deviation (recorded below,
# 256x256: ~1.5e-3) with headroom for the fp32 accumulation of the GPU
FRAME_BAR = 6e-3


def test_identity_hook_reproduces_the_oracle():
    from oracle import net_oracle
    f = synth.make_frame(64, 96, 1)
    a = net_oracle.NetOracle(style="candy", dtype=torch.float64).run_image(f)
    b = net_oracle.NetOracle(style="candy", dtype=torch.float64, operand_round=fo.Fp16Round(False)).run_image(f)
    assert np.array_equal(a, b)


def test_weights_are_the_packed_hi_halves():
    w = synth.make_weights(synth.DEFAULT_ARCH, "candy")
    for name in ("l0.weight", "l3.c1.weight", "l8.weight", "l10.weight"):
        if name not in w:
            continue
        a = w[name].astype(np.float64)
        h = fo.packed_hi_weights(w[name], transposed=name.startswith("l8"))
        assert not np.array_equal(h, a)
        assert np.abs(h - a).max() <= np.abs(a).max() * 2.0 ** -11


def test_expected_frame_error_of_the_mode():
    from oracle import net_oracle
    H, W = 256, 256
    f = synth.make_frame(H, W, 1)
    exact = net_oracle.NetOracle(style="candy", dtype=torch.float64).run_image(f)
    emu = fo.fp16_oracle(style="candy").run_image(f)
    d = float(np.abs(emu - exact).max())
    print(f"\nfp16 mode emulator vs fp64 at {W}x{H}: max-abs {d:.3e} ({d * 255:.2f} 8-bit levels)")
    assert 1e-5 < d < FRAME_BAR / 2, d
