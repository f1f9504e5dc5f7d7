"""The bicubic image.scale reading of tests/scale_oracle.py (DESIGN.md §8), pinned by properties that do not depend on it:
constants stay constant, planes linear in x and y are reproduced everywhere (linearly extrapolated borders; clamped ones would
fail), quadratics are reproduced wherever all four taps lie inside the line (Keys, a = -1/2), an equal size is a copy, the last
sample is the last source sample, and sides of 1 are refused.  No GPU."""
import ctypes as C

import numpy as np
import pytest

import scale_oracle as so

SIZE_PAIRS = [(7, 3), (3, 7), (97, 48), (48, 97)]


def grid_positions(n, m):
    """the oracle's own fp32 sample positions along a line of n -> m samples, as float64 (the last one is n - 1)"""
    if m == n:
        return np.arange(n, dtype=np.float64)
    i, f = so.positions(n, m)
    return np.concatenate([(i.astype(np.float32) + f).astype(np.float64), [n - 1.0]])


@pytest.mark.parametrize("n,m", SIZE_PAIRS)
def test_constant_planes_stay_constant(n, m):
    for v in (0.0, 1.0, -0.37, 123.456):
        src = np.full((2, n, n + 3), v, np.float32)
        v = float(src[0, 0, 0])
        out = so.image_scale_bicubic(src, m, m + 5)
        assert out.shape == (2, m, m + 5)
        assert np.abs(out - v).max() <= 1e-12 * max(1.0, abs(v))


@pytest.mark.parametrize("n,m", SIZE_PAIRS)
def test_linear_planes_are_reproduced_everywhere(n, m):
    """a + b x + c y at the fp32 positions, the outer samples included: the border taps 2*p1 - p2 continue the line"""
    Hin, Win, Hout, Wout = n, n + 4, m, m + 2
    y, x = np.mgrid[0:Hin, 0:Win].astype(np.float64)
    for a, b, c in ((0.5, 0.25, -0.125), (-3.0, 1.5, 2.0)):
        src = a + b * x + c * y  # exact in fp32 for these coefficients
        assert np.array_equal(src.astype(np.float32), src)
        out = so.image_scale_bicubic(src.astype(np.float32), Hout, Wout)
        Y, X = np.meshgrid(grid_positions(Hin, Hout), grid_positions(Win, Wout), indexing="ij")
        want = a + b * X + c * Y
        scale = np.abs(src).max()
        assert np.abs(out - want).max() <= 1e-12 * scale


def test_clamped_borders_would_fail_the_linear_case():
    """the linear case really tests the border rule: clamping p0 = p1 at i = 0 moves the first interpolated samples"""
    n, m = 7, 3 * 7
    line = np.arange(n, dtype=np.float64)
    i, f32 = so.positions(n, m)
    f = f32.astype(np.float64)
    p1, p2 = line[i], line[i + 1]
    p0 = np.where(i > 0, line[np.maximum(i - 1, 0)], p1)  # clamped
    p3 = np.where(i + 2 < n, line[np.minimum(i + 2, n - 1)], p2)
    clamped = p1 + 0.5 * f * ((p2 - p0) + f * ((2 * p0 - 5 * p1 + 4 * p2 - p3) + f * (3 * (p1 - p2) + p3 - p0)))
    assert np.abs(clamped - grid_positions(n, m)[:-1]).max() > 1e-3


@pytest.mark.parametrize("n,m", SIZE_PAIRS)
def test_quadratics_are_reproduced_inside(n, m):
    """q(x) = a + b x + c x^2 along x (constant along y): exact at output samples whose four taps 1 <= i <= n - 3 lie inside"""
    Hin = 5
    x = np.arange(n, dtype=np.float64)
    q = lambda t: 0.75 - 0.5 * t + 0.0625 * t * t
    src = np.broadcast_to(q(x), (Hin, n)).astype(np.float32)
    assert np.array_equal(src[0].astype(np.float64), q(x))
    out = so.image_scale_bicubic(src, Hin, m)
    i, _ = so.positions(n, m)
    inside = np.nonzero((i >= 1) & (i <= n - 3))[0]
    if n < 4:  # a line of 3 has no sample with four taps inside
        assert len(inside) == 0
        return
    assert len(inside) > 0
    X = grid_positions(n, m)[inside]
    assert np.abs(out[:, inside] - q(X)[None]).max() <= 1e-12 * np.abs(src).max()


def test_equal_size_is_a_copy():
    src = np.random.default_rng(1).uniform(-0.2, 1.2, (3, 13, 17)).astype(np.float32)
    assert np.array_equal(so.image_scale_bicubic(src, 13, 17), src)
    # one side equal: that pass copies, so every row is the x pass alone
    rows = so.image_scale_bicubic(src, 13, 40)
    cols = so.image_scale_bicubic(src, 31, 17)
    for k in range(3):
        for r in range(13):
            assert np.array_equal(rows[k, r], so.image_scale_bicubic(src[k, r][None].repeat(2, 0), 2, 40)[0])
        for c in range(17):
            assert np.array_equal(cols[k, :, c], so.image_scale_bicubic(src[k, :, c][None].repeat(2, 0), 2, 31)[0])


@pytest.mark.parametrize("n,m", SIZE_PAIRS + [(1280, 640), (640, 1280), (720, 1441)])
def test_last_sample_is_the_last_source_sample(n, m):
    src = np.random.default_rng(n * 7 + m).uniform(-0.2, 1.2, (2, n)).astype(np.float32)
    out = so.image_scale_bicubic(src, 2, m)
    assert np.array_equal(out[:, -1], src[:, -1].astype(np.float64))
    out = so.image_scale_bicubic(src.T.copy(), m, 2)
    assert np.array_equal(out[-1], src[:, -1].astype(np.float64))
    # the fp32 positions never reach the last interval's end before d = m - 1
    i, f = so.positions(n, m)
    assert i.max() <= n - 2 and (f >= 0).all() and (f < 1).all()


def test_fp32_two_pass_form_is_close_to_fp64():
    src = np.random.default_rng(2).uniform(-0.2, 1.2, (3, 97, 75)).astype(np.float32)
    for Hout, Wout in ((48, 37), (194, 150), (97, 150)):
        ref = so.image_scale_bicubic(src, Hout, Wout)
        assert np.abs(so.image_scale_bicubic_fp32(src, Hout, Wout) - ref).max() <= 2e-6 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("shape_in,shape_out", [((1, 5), (3, 5)), ((5, 1), (5, 3)), ((5, 5), (1, 5)), ((5, 5), (5, 1))])
def test_sides_of_one_are_refused(shape_in, shape_out):
    with pytest.raises(ValueError):
        so.image_scale_bicubic(np.zeros(shape_in, np.float32), *shape_out)
    from fav_b200 import _lib

    fake = C.c_void_p(16)  # never dereferenced: the sizes are refused before anything is launched
    assert _lib.lib.fav_image_scale_bicubic(fake, fake, 3, *shape_in, *shape_out, None) == _lib.FAV_ERR_INVALID
    assert "every size must be 2" in _lib.last_error()
