"""Pins the warp against the REFERENCE ITSELF: outputs of the reference's own CUDA kernel (stnbdhw/BilinearSamplerBDHW.cu:48-109,
compiled for sm_90a behind oracle/ref_warp/harness.cu, original (32,16) block / (C, H*ceil(W/512), B) grid), recorded on an
H100 by tests/golden/make_warp_golden.py into tests/golden/refwarp_cases.npz and warp_ref.npz, vs the product's
fav_bilinear_sampler_bdhw_update_output / fused temporal input and vs the C oracle.  Bar: BIT-EXACT (SHA-256 of every
output) at every BASELINE.json config shape, real and stress flows, and on the committed vectors."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_warp_golden as mwg  # noqa: E402


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "refwarp_cases.npz"))


@pytest.mark.parametrize("shape", mwg.REF_SHAPES)
def test_product_warp_equals_reference_kernel(gold, shape):
    from fav_b200 import utils

    H, W = shape
    img, flows = mwg.shape_inputs(H, W)
    for name, flow in flows.items():
        g = utils.warp_image(T(img), T(flow)).cpu().numpy()
        key = f"{H}x{W}_{name}"
        if mwg.digest(g) != str(gold[key + "_sha"]):
            want, got = gold[key + "_sample"], g.reshape(-1)[mwg.sample_index(g.size)]
            pytest.fail(f"{shape} {name}: output differs from the reference kernel's; {int((want != got).sum())} of "
                        f"{want.size} sampled values differ")


def test_reference_kernel_batch_channels_and_output_size(gold):
    from fav_b200 import stn

    img, grid = mwg.batch_inputs()
    assert np.array_equal(stn.BilinearSamplerBDHW().forward((T(img), T(grid))).cpu().numpy(), gold["batch"])
    g = torch.full((1, 2, 20, 28), 99999.0, device="cuda")  # sentinel flow of vr_helper.lua:10
    assert float(np.abs(gold["sentinel"]).max()) == 0.0
    assert np.array_equal(stn.BilinearSamplerBDHW().forward((T(img[:1]), g)).cpu().numpy(), gold["sentinel"])


def test_fused_temporal_input_prior_equals_reference_kernel_composition(gold):
    """in[3:6] of the fused kernel == preprocess(reference-kernel warp) * cert composed with torch ops in the
    reference's op order (core.lua:166-167), bit for bit."""
    from fav_b200 import _lib

    c, p, flow, cert = (T(a) for a in mwg.prior_inputs())
    H, W = c.shape[-2:]
    out = torch.empty((7, H, W), device="cuda")
    _lib.check(_lib.lib.fav_temporal_input(_lib.dptr(c), _lib.dptr(p), _lib.dptr(flow), _lib.dptr(cert), None, None,
                                           _lib.dptr(out), H, W, 0, _lib.stream_ptr()))
    assert mwg.digest(out[3:6].cpu().numpy()) == str(gold["prior_360x640_sha"])


def test_oracle_and_product_reproduce_committed_reference_vectors():
    """tests/golden/warp_ref.npz was written by the reference kernel (make_warp_golden.py)."""
    from fav_b200 import stn
    from oracle import pyoracle

    gold = np.load(os.path.join(ROOT, "tests", "golden", "warp_ref.npz"))
    for case in mwg.WARP_CASES:
        img, flow = mwg.warp_inputs(case)
        assert np.array_equal(stn.BilinearSamplerBDHW().forward((T(img), T(flow))).cpu().numpy(), gold[case[0]]), case[0]
        assert np.array_equal(pyoracle.warp_bdhw(img, flow), gold[case[0]]), case[0]
