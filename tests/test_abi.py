"""The C-ABI shared library loads and exports every symbol include/fav.h declares; without a GPU every compute
entry point fails loudly (no CPU fallback)."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "fav.h")).read()
    return sorted(set(re.findall(r"FAV_API\s+[\w\s\*]+?\b(fav_\w+)\s*\(", txt)))


def test_header_symbols_exported():
    from fav_b200 import _lib

    syms = header_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(_lib.lib, s), f"{s} declared in fav.h but not exported by libfav_b200.so"
    # and the Python binding table covers exactly the header
    assert sorted(_lib.SIGNATURES) == syms


def test_every_declaration_cites_the_reference():
    txt = open(os.path.join(ROOT, "include", "fav.h")).read()
    assert txt.count(".cu:") + txt.count(".lua:") + txt.count(".cpp:") >= 15


def test_grad_entry_points_raise_like_the_reference():
    from fav_b200 import _lib

    assert _lib.lib.fav_bilinear_sampler_bdhw_update_grad_input() == _lib.FAV_ERR_NOT_IMPLEMENTED
    assert "Not implemented" in _lib.last_error()  # BilinearSamplerBDHW.cu:173
    assert _lib.lib.fav_bilinear_sampler_bdhw_update_grad_input_only_grid() == _lib.FAV_ERR_NOT_IMPLEMENTED


def test_argument_validation_without_compute():
    import ctypes as C

    from fav_b200 import _lib

    z = _lib.i64x4([1, 3, 4, 4])
    bad = _lib.i64x4([1, 3, 4, 4])  # grids:size(2) must be 2
    fake = C.c_void_p(16)
    st = _lib.lib.fav_bilinear_sampler_bdhw_update_output(fake, z, z, fake, bad, z, fake, z, 0, None)
    assert st == _lib.FAV_ERR_INVALID and "size(2)" in _lib.last_error()
    assert _lib.lib.fav_min_filter(fake, fake, 1, 4, 4, 4, None) == _lib.FAV_ERR_INVALID  # even r


def test_arch_parser_and_param_table():
    from fav_b200 import models_video, synth

    net = models_video.StyleNet(synth.DEFAULT_ARCH)
    shapes = net.param_shapes()
    w = synth.make_weights(synth.DEFAULT_ARCH, "candy")
    assert set(shapes) == set(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(shapes[k]), k
    with pytest.raises(Exception) as e:
        models_video.StyleNet("c9s1-32,X5,c9s1-3")
    assert "not supported" in str(e.value)
    from fav_b200 import _lib

    # one stride-2 layer, two upsampling ones: the net would return a 2H x 2W image, past the [3][H][W] output frame
    with pytest.raises(_lib.FavError) as e:
        models_video.StyleNet("c9s1-32,d64,R64,u32,u8,c9s1-3")
    assert e.value.status == _lib.FAV_ERR_UNSUPPORTED and "resizes the frame by 2" in str(e.value)


def test_no_cpu_fallback_without_device():
    import torch

    from fav_b200 import _lib, models_video, synth

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = models_video.StyleNet()
    with pytest.raises(_lib.FavError) as e:
        net.load_state(synth.make_weights())
    assert e.value.status == _lib.FAV_ERR_NO_DEVICE
    import ctypes as C

    fake = C.c_void_p(16)
    assert _lib.lib.fav_vgg_preprocess(fake, fake, 1, 4, 4, None) == _lib.FAV_ERR_NO_DEVICE
    assert "no CPU fallback" in _lib.last_error()


def test_flo_reader_matches_oracle(tmp_path):
    from fav_b200 import flowFileLoader, synth
    from oracle import pyoracle

    uv = synth.make_backward_flow(37, 53, 2)
    p = str(tmp_path / "a.flo")
    synth.write_flo(p, uv)
    lua = flowFileLoader.load(p)  # [dy, dx]  (flowFileLoader.lua:31-32)
    assert np.array_equal(lua, pyoracle.flo_read(p, 0)) and np.array_equal(lua[0], uv[1]) and np.array_equal(lua[1], uv[0])
    chk = flowFileLoader.load(p, layout=1)
    assert np.array_equal(chk, pyoracle.flo_read(p, 1)) and np.array_equal(chk, uv)
    open(str(tmp_path / "trunc.flo"), "wb").write(open(p, "rb").read()[:100])
    with pytest.raises(Exception):
        flowFileLoader.load(str(tmp_path / "trunc.flo"))
    with pytest.raises(Exception):
        flowFileLoader.load(str(tmp_path / "missing.flo"))
    # hostile header (2^30 x 2^30) and a file that outgrew the caller's buffer: FAV_ERR_IO, never an exception / overflow
    import struct

    from fav_b200 import _lib

    open(str(tmp_path / "huge.flo"), "wb").write(struct.pack("<fii", 202021.25, 1 << 30, 1 << 30) + b"\0" * 64)
    with pytest.raises(_lib.FavError) as e:
        flowFileLoader.load(str(tmp_path / "huge.flo"))
    assert e.value.status == _lib.FAV_ERR_IO
    small = np.empty((2, 10, 10), np.float32)
    with pytest.raises(_lib.FavError) as e:
        flowFileLoader.load(p, out=small)
    assert e.value.status == _lib.FAV_ERR_IO


def test_pnm_readers(tmp_path):
    """image.load(ppm|pgm) = byte / 255 (fast_artistic_video.lua:95,103) and readFromPPM's 0..255 planes with comments."""
    import ctypes as C

    from fav_b200 import _lib, synth

    H, W = 13, 21
    img = synth.make_frame(H, W, 4)
    p = str(tmp_path / "f.ppm")
    synth.write_ppm(p, img)
    u8 = np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8)
    w_, h_, c_ = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib.fav_pnm_read_header(p.encode(), C.byref(w_), C.byref(h_), C.byref(c_)))
    assert (w_.value, h_.value, c_.value) == (W, H, 3)
    out = np.empty((3, H, W), np.float32)
    _lib.check(_lib.lib.fav_pnm_read_f32(p.encode(), out.ctypes.data_as(C.c_void_p), out.size, C.c_float(255.0)))
    assert np.array_equal(out, u8.astype(np.float32) / np.float32(255.0))
    g = (np.random.default_rng(0).uniform(size=(H, W)) > 0.3).astype(np.uint8) * 255
    pg = str(tmp_path / "c.pgm")
    open(pg, "wb").write(b"P5\n# a comment line\n%d %d\n255\n" % (W, H) + g.tobytes())
    outg = np.empty((1, H, W), np.float32)
    _lib.check(_lib.lib.fav_pnm_read_f32(pg.encode(), outg.ctypes.data_as(C.c_void_p), outg.size, C.c_float(1.0)))
    assert np.array_equal(outg[0], g.astype(np.float32))
    assert _lib.lib.fav_pnm_read_f32(pg.encode(), outg.ctypes.data_as(C.c_void_p), 5, C.c_float(1.0)) == _lib.FAV_ERR_IO


def test_raw_payload_readers(tmp_path):
    """fav_pnm_read_u8 / fav_flo_read_raw: the payloads as stored (for the GPU-side conversions of
    fav_session_run_frame_bytes), sizes returned, capacity enforced, hostile headers rejected."""
    import ctypes as C
    import struct

    from fav_b200 import _lib, synth

    H, W = 9, 14
    img = synth.make_frame(H, W, 2)
    p = str(tmp_path / "f.ppm")
    synth.write_ppm(p, img)
    u8 = np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8)  # CHW
    out = np.zeros((H, W, 3), np.uint8)
    w_, h_, c_ = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib.fav_pnm_read_u8(p.encode(), out.ctypes.data_as(C.c_void_p), out.size, C.byref(w_), C.byref(h_), C.byref(c_)))
    assert (w_.value, h_.value, c_.value) == (W, H, 3) and np.array_equal(out, u8.transpose(1, 2, 0))
    assert _lib.lib.fav_pnm_read_u8(p.encode(), out.ctypes.data_as(C.c_void_p), out.size - 1, C.byref(w_), C.byref(h_), C.byref(c_)) == _lib.FAV_ERR_IO
    uv = synth.make_backward_flow(H, W, 3)
    pf = str(tmp_path / "b.flo")
    synth.write_flo(pf, uv)
    raw = np.zeros((H, W, 2), np.float32)
    _lib.check(_lib.lib.fav_flo_read_raw(pf.encode(), raw.ctypes.data_as(C.c_void_p), raw.size, C.byref(w_), C.byref(h_)))
    assert (w_.value, h_.value) == (W, H) and np.array_equal(raw[..., 0], uv[0]) and np.array_equal(raw[..., 1], uv[1])
    assert _lib.lib.fav_flo_read_raw(pf.encode(), raw.ctypes.data_as(C.c_void_p), raw.size - 1, C.byref(w_), C.byref(h_)) == _lib.FAV_ERR_IO
    open(str(tmp_path / "huge.flo"), "wb").write(struct.pack("<fii", 202021.25, 1 << 30, 1 << 30) + b"\0" * 64)
    assert _lib.lib.fav_flo_read_raw(str(tmp_path / "huge.flo").encode(), raw.ctypes.data_as(C.c_void_p), raw.size, C.byref(w_), C.byref(h_)) == _lib.FAV_ERR_IO
    open(str(tmp_path / "trunc.ppm"), "wb").write(b"P6\n%d %d\n255\n" % (W, H) + b"\0" * 10)
    assert _lib.lib.fav_pnm_read_u8(str(tmp_path / "trunc.ppm").encode(), out.ctypes.data_as(C.c_void_p), out.size, C.byref(w_), C.byref(h_), C.byref(c_)) == _lib.FAV_ERR_IO


def test_png_writer_round_trip(tmp_path):
    """fav_png_write (image.save of an 8-bit image): decoded by an independent PNG reader (PIL) the pixels are identical, for one
    band and for concurrent deflate bands, RGB and gray, every compression mode."""
    import ctypes as C

    from PIL import Image

    from fav_b200 import _lib

    rng = np.random.default_rng(3)
    for (H, W, Cn, nt, lvl) in [(7, 5, 3, 1, 1), (64, 33, 1, 4, 1), (1100, 1000, 3, 3, 1), (300, 200, 3, 4, 0), (300, 200, 3, 3, 6)]:
        yy, xx = np.mgrid[0:H, 0:W]
        img = np.stack([(128 + 100 * np.sin(xx / 37 + c) * np.cos(yy / 23) + rng.normal(0, 12, (H, W))).clip(0, 255) for c in range(Cn)], -1)
        img = np.ascontiguousarray(img.astype(np.uint8))
        p = str(tmp_path / "a.png")
        _lib.check(_lib.lib.fav_png_write(p.encode(), img.ctypes.data_as(C.c_void_p), W, H, Cn, lvl, nt))
        back = np.asarray(Image.open(p))
        assert np.array_equal(back if Cn == 3 else back[..., None], img), (H, W, Cn, nt, lvl)
    assert _lib.lib.fav_png_write(str(tmp_path / "no" / "dir.png").encode(), img.ctypes.data_as(C.c_void_p), W, H, Cn, 1, 1) == _lib.FAV_ERR_IO
    assert _lib.lib.fav_png_write(b"x.png", img.ctypes.data_as(C.c_void_p), W, H, 2, 1, 1) == _lib.FAV_ERR_INVALID
