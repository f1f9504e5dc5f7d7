"""The fp64 restatement of the VR driver's -evaluate (tests/vr_eval_oracle.py) against an independent formulation with scipy,
the reference's seam-metric quirks, and the refusal of unequal overlaps (CPU only)."""
import math

import numpy as np
import pytest
from scipy import ndimage, signal

import vr_eval_oracle as ve
from oracle import vr_oracle


def masks(S, ov, r=7):
    ref = vr_oracle.VRRef(S, S, ov, ov, 3, 8, 8)
    ev = ve.VREval(ref, None, None, None, reliable_map_min_filter=r)
    return {"left": ev.mask_left, "right": ev.mask_right, "left_right": ev.mask_left_right, "all": ev.mask_all}


def scipy_metric(img, mask):
    """evaluate_gradient written independently: 'valid' convolutions, a 3x3 maximum filter whose padding is -inf, and the
    ratios as masked means over full means."""
    d = img.astype(np.float64)
    kx, ky = np.array([[-1.0, 0.0, 1.0]]), np.array([[-1.0], [0.0], [1.0]])
    gx = np.max([np.abs(signal.convolve2d(d[c], kx, "valid")) for c in range(3)], axis=0)
    gy = np.max([np.abs(signal.convolve2d(d[c], ky, "valid")) for c in range(3)], axis=0)
    m = mask[0].astype(np.float64)
    mx = ndimage.maximum_filter(np.abs(signal.convolve2d(m, kx, "valid")), size=3, mode="constant", cval=-np.inf)
    my = ndimage.maximum_filter(np.abs(signal.convolve2d(m, ky, "valid")), size=3, mode="constant", cval=-np.inf)
    sums = [gx.sum(), gy.sum(), mx.sum(), my.sum(), (gx * mx).sum(), (gy * my).sum()]
    with np.errstate(divide="ignore", invalid="ignore"):
        rx = ((gx * mx).sum() / mx.sum()) / gx.mean()
        ry = ((gy * my).sum() / my.sum()) / gy.mean()
        rm = (rx * mx.sum() + ry * my.sum()) / (mx.sum() + my.sum())
    return sums, (float(rx), float(ry), float(rm))


def close(a, b, rel=1e-12):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= rel * max(abs(a), abs(b))


@pytest.mark.parametrize("S", [64, 100, 128])
@pytest.mark.parametrize("ov", [20, 32])
def test_gradient_metric_matches_independent_formulation(S, ov):
    rng = np.random.default_rng(S + ov)
    for k, (name, m) in enumerate(masks(S, ov).items()):
        img = rng.uniform(-0.2, 1.2, size=(3, S, S)).astype(np.float32)
        sums = ve.gradient_sums(img, m)
        ref_sums, ref_ratios = scipy_metric(img, m)
        assert all(close(a, b) for a, b in zip(sums, ref_sums)), (name, sums, ref_sums)
        got = ve.evaluate_gradient(img, m)
        assert all(close(a, b) for a, b in zip(got, ref_ratios)), (name, got, ref_ratios)
        assert sums[2] > 0 and sums[3] > 0 and all(np.isfinite(got)), name  # every real mask has an edge to measure


def test_gradient_metric_of_an_edgeless_mask_is_nan():
    img = np.random.default_rng(0).uniform(size=(3, 40, 52)).astype(np.float32)
    for m in (np.zeros((1, 40, 52), np.float32), np.ones((1, 40, 52), np.float32)):
        sums = ve.gradient_sums(img, m)
        assert sums[2] == sums[3] == sums[4] == sums[5] == 0.0
        assert all(math.isnan(v) for v in ve.evaluate_gradient(img, m))  # 0/0 as in Lua
        assert all(math.isnan(v) for v in scipy_metric(img, m)[1])
    # a flat face against a real mask: masked / full = 0/0 as well
    m = masks(40, 20)["left"]
    flat = np.full((3, 40, 40), 0.3, np.float32)
    assert all(math.isnan(v) for v in ve.evaluate_gradient(flat, m))


def test_driver_ratios_match_the_restatement():
    from fav_b200 import vr

    img = np.random.default_rng(1).uniform(size=(3, 64, 64)).astype(np.float32)
    for m in (masks(64, 20)["all"], np.zeros((1, 64, 64))):
        sums = ve.gradient_sums(img, m)
        a, b = vr.gradient_ratios(sums, 64, 64), ve.gradient_ratios(sums, 64, 64)
        assert all(close(x, y, 0.0) for x, y in zip(a, b)), (a, b)
    # x/0 is inf, not an exception
    assert vr.gradient_ratios([0.0, 1.0, 1.0, 1.0, 1.0, 1.0], 8, 8)[0] == math.inf


def test_seam_metric_quirks():
    rng = np.random.default_rng(2)
    S, ov = 64, 20
    faces = {k: rng.uniform(size=(3, S, S)).astype(np.float32) for k in range(1, 7)}
    t = {k: ve.trim(v, ov, ov) for k, v in faces.items()}
    assert t[1].shape == (3, S - ov, S - ov)
    # evaluate_edge_top never reads its first argument, and its 'top' term compares a row with itself
    assert ve.evaluate_edge_top(t[1], t[5], "top") == 0.0
    for edge in ("right", "left", "bottom"):
        v = ve.evaluate_edge_top(t[2], t[5], edge)
        assert v == ve.evaluate_edge_top(t[3], t[5], edge) == ve.evaluate_edge_top(None, t[5], edge) and v > 0
    five = t[5].astype(np.float64)
    assert ve.evaluate_edge_top(None, t[5], "left") == np.mean((five[:, 0, :] - five[:, :, 0]) ** 2)
    assert ve.evaluate_edge_top(None, t[5], "right") == np.mean((five[:, 0, :] - five[:, ::-1, -1]) ** 2)
    assert ve.evaluate_edge_top(None, t[5], "bottom") == np.mean((five[:, 0, :] - five[:, -1, :]) ** 2)
    assert ve.evaluate_edge(t[1], t[2], "left") == np.mean((t[1][:, :, 0].astype(np.float64) - t[2][:, :, -1]) ** 2)
    # unequal overlaps: the trimmed face is not square, and the mode-4 criterion compares slices of different lengths
    with pytest.raises(ValueError):
        ve.evaluate_edge_top(None, ve.trim(faces[5], 20, 32), "left")


def test_vr_evaluate_refuses_unequal_overlaps():
    from fav_b200 import _lib, vr

    with pytest.raises(_lib.FavError) as e:
        vr.main(["-input_pattern", "x_%d_%d.ppm", "-create_inconsistent", "-evaluate", "-overlap_pixel_w", "20",
                 "-overlap_pixel_h", "32"])
    assert e.value.status == _lib.FAV_ERR_INVALID and "overlap_pixel_w == overlap_pixel_h" in e.value.message


def test_vr_parser_declares_the_evaluation_options():
    from fav_b200 import vr

    opt = vr.build_parser().parse_args([])
    assert (opt.evaluation_file, opt.style_weights, opt.style_image, opt.style_layers, opt.content_layers, opt.content_weights,
            opt.style_image_size, opt.style_target_type, opt.reliable_map_min_filter) == (
        "evaluation.txt", "5.0", "", "4,9,16,23", "16", "1.0", 256, "gram", 7)
    assert not (opt.no_consistency_eval or opt.backward_eval or opt.invert_occlusions_eval or opt.fix_occlusions_eval)
    assert opt.flow_pattern_eval == opt.occlusions_pattern_eval == ""


def test_fix_occlusions_rule():
    """:117-128 tests the displacement itself against [0, H] x [0, W], not the warped position."""
    H, W = 5, 7
    flow = np.zeros((2, H, W), np.float32)
    flow[0, 0, 0], flow[1, 1, 1], flow[0, 2, 2], flow[1, 3, 3], flow[0, 4, 4] = -0.5, W + 0.5, H + 0.1, -1e-3, H
    cert = np.ones((1, H, W), np.float32)
    ve.fix_occlusions(flow, cert)
    zeroed = {(int(y), int(x)) for y, x in zip(*np.nonzero(cert[0] == 0))}
    assert zeroed == {(0, 0), (1, 1), (2, 2), (3, 3)}
