"""Generates the 4-argument-mode golden masks for the edge cases of the structure term (run where oracle/_ref is built):

  structure_const_64x96.npz : a constant frame -- every corner is 0, the average is 0 and the structure term is 4/0 * 0 (NaN):
                              the threshold is NaN, `lhs >= threshold` never holds, and every pixel whose flow lands inside
                              the frame is reliable
  structure_16x16.npz       : a 16 x 16 frame (one sub-chunk of the exact average, the smallest frame a session takes)

Each holds the {0,255} mask written by the reference's own consistencyChecker binary in 4-argument mode (oracle/_ref/, compiled
unmodified by oracle/Makefile).  Inputs are regenerated from seeds by structure_inputs(); only the masks are stored.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402

from fav_b200 import synth  # noqa: E402
from oracle import pyoracle  # noqa: E402

STRUCTURE_CASES = {"const_64x96": (64, 96, 2, 0.6, 6), "16x16": (16, 16, 2, 0.6, 7)}


def structure_inputs(name):
    """bw, fw (u,v), frame in [0,1] and its 0..255 planes of one case."""
    H, W, idx, sigma, seed = STRUCTURE_CASES[name]
    bw, fw, fr, img255 = make_golden.consistency_inputs(H, W, idx, sigma, seed)
    if name.startswith("const"):
        fr = np.full_like(fr, 0.4)
        img255 = np.clip(np.rint(fr * 255.0), 0, 255).astype(np.float32)
    return bw, fw, fr, img255


def main():
    assert os.path.exists(pyoracle.REF_CHECKER), "build oracle/_ref first (make -C oracle ref)"
    for name in STRUCTURE_CASES:
        bw, fw, fr, _ = structure_inputs(name)
        d = tempfile.mkdtemp()
        synth.write_flo(d + "/bw.flo", bw); synth.write_flo(d + "/fw.flo", fw); synth.write_ppm(d + "/f.ppm", fr)
        pyoracle.run_ref_checker(d + "/bw.flo", d + "/fw.flo", d + "/r4.pgm", d + "/f.ppm")
        r4 = synth.read_pgm(d + "/r4.pgm")
        assert set(np.unique(r4)) <= {0, 255}
        np.savez_compressed(os.path.join(HERE, f"structure_{name}.npz"), ref4=np.packbits(r4 == 255), shape=np.array(r4.shape))
        print(name, "zeros", (r4 == 0).sum())


if __name__ == "__main__":
    main()
