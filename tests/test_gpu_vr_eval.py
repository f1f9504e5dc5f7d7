"""-evaluate of the VR driver on the GPU: fav_vr_eval_gradient against the fp64 restatement (tests/vr_eval_oracle.py), and
`vr.main -evaluate` against the driver restatement with the evaluation hook, over every option of the evaluation."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import vr_eval_oracle as ve
from fav_b200 import _lib, percep, synth, t7, vr
from oracle import percep_oracle, vr_oracle

pytestmark = pytest.mark.gpu

GRAD_REL = 1e-12   # six double sums of fp32 inputs, reordered
LOSS_BAR = 1e-4    # relative, the perceptual-loss bar of tests/test_gpu_percep.py


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(a, b, rel):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= rel * max(abs(a), abs(b))


def kernel_sums(face, mask):
    H, W = face.shape[-2:]
    out = torch.full((6,), -1.0, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib.fav_vr_eval_gradient(_lib.dptr(face), _lib.dptr(mask), H, W, _lib.dptr(out), _lib.stream_ptr()))
    return out


def real_mask(S, ov, which):
    ref = vr_oracle.VRRef(S, S, ov, ov, 3, 8, 8)
    ev = ve.VREval(ref, None, None, None)
    return {"left": ev.mask_left, "right": ev.mask_right, "left_right": ev.mask_left_right, "all": ev.mask_all}[which]


@pytest.mark.parametrize("H,W,ov,which", [(64, 64, 20, "left"), (64, 64, 20, "left_right"), (100, 100, 32, "all"),
                                          (100, 100, 20, "right"), (517, 389, None, None), (2048, 2048, 128, "all")])
def test_eval_gradient_kernel_vs_fp64(H, W, ov, which):
    rng = np.random.default_rng(H + W)
    face = rng.uniform(-0.2, 1.2, size=(3, H, W)).astype(np.float32)
    if which is None:  # non-square and odd: a smooth mask with flat, ramped and hard edges
        yy, xx = np.mgrid[0:H, 0:W]
        mask = np.clip(np.sin(xx / 23.0) * np.cos(yy / 17.0) * 2.0, 0.0, 1.0).astype(np.float32)[None]
        mask[:, 100:140, :] = (rng.uniform(size=(40, W)) > 0.5)
    else:
        mask = real_mask(H, ov, which).astype(np.float32)
    ref = ve.gradient_sums(face, mask)
    tf, tm = cuda(face), cuda(mask[0])
    a = kernel_sums(tf, tm)
    b = kernel_sums(tf, tm)
    assert torch.equal(a, b), "two calls differ"
    got = a.tolist()
    errs = [abs(g - r) / abs(r) if r else abs(g) for g, r in zip(got, ref)]
    print(f"\n{H}x{W} {which}: sums {got}, max rel err {max(errs):.2e}")
    assert max(errs) <= GRAD_REL, (got, ref)
    assert all(same(x, y, GRAD_REL) for x, y in zip(vr.gradient_ratios(got, H, W), ve.gradient_ratios(ref, H, W)))


def test_eval_gradient_refusals():
    f, m = torch.zeros((3, 8, 8), device="cuda"), torch.zeros((8, 8), device="cuda")
    s = torch.zeros(6, dtype=torch.float64, device="cuda")
    st = _lib.stream_ptr()
    for H, W in ((2, 8), (8, 2), (0, 0), (-1, 5)):
        assert _lib.lib.fav_vr_eval_gradient(_lib.dptr(f), _lib.dptr(m), H, W, _lib.dptr(s), st) == _lib.FAV_ERR_INVALID
    assert _lib.lib.fav_vr_eval_gradient(None, _lib.dptr(m), 8, 8, _lib.dptr(s), st) == _lib.FAV_ERR_INVALID
    assert _lib.lib.fav_vr_eval_gradient(_lib.dptr(f), None, 8, 8, _lib.dptr(s), st) == _lib.FAV_ERR_INVALID
    assert _lib.lib.fav_vr_eval_gradient(_lib.dptr(f), _lib.dptr(m), 8, 8, None, st) == _lib.FAV_ERR_INVALID
    assert "null" in _lib.last_error()
    # the smallest face: one row of gy, one column of gx
    face = np.random.default_rng(0).uniform(size=(3, 3, 3)).astype(np.float32)
    mask = np.random.default_rng(1).uniform(size=(1, 3, 3)).astype(np.float32)
    got, ref = kernel_sums(cuda(face), cuda(mask[0])).tolist(), ve.gradient_sums(face, mask)
    assert all(same(g, r, GRAD_REL) for g, r in zip(got, ref)), (got, ref)


# ---- the driver ---------------------------------------------------------------------------------------------------------
class FakeGpuNet:
    """exact fp32 elementwise ops, the same on both sides, so the driver logic is checked independently of the network"""

    def run_image(self, img, fill=None):
        return (img * 0.5).contiguous()

    def run_next_image(self, img, prev, flow, cert, fill=None, flow_mask=None, border_mode=0):
        m = cert if flow_mask is None else torch.minimum(cert, flow_mask)
        return (img * 0.25 + (prev * m) * 0.75).contiguous()


class FakeRefNet:
    def run_image(self, img):
        return (img * np.float32(0.5)).astype(np.float32)

    def run_next_image_prior(self, img, prior, cert, fmask):
        m = cert if fmask is None else np.minimum(cert, fmask)
        return ((img * np.float32(0.25)).astype(np.float32) + ((prior * m[None]).astype(np.float32) * np.float32(0.75))
                .astype(np.float32)).astype(np.float32)


def write_clip(d, S, n, prefix="", seed0=0):
    """n VR frames x 6 faces as PPMs, per-face backward flows and occlusion PGMs; returns what the reference would load"""
    frames, flows, certs = [], [], []
    for f in range(1, n + 1):
        fr, fl, ce = {}, {}, {}
        for face in range(1, 7):
            if not prefix:
                img = synth.make_frame(S, S, 10 * f + face + seed0)
                synth.write_ppm(f"{d}/in_{f:03d}_{face}.ppm", img)
                fr[face] = np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8).astype(np.float32) / 255.0
            if f >= 2:
                bw = synth.make_backward_flow(S, S, face + f + 7 * seed0)
                synth.write_flo(f"{d}/{prefix}bw_{f}_{f - 1}_{face}.flo", bw)
                fl[face] = synth.checker_to_lua(bw)
                rel = (np.random.default_rng(100 * f + face + seed0).uniform(size=(S, S)) > 0.1).astype(np.uint8) * 255
                with open(f"{d}/{prefix}rel_{f}_{f - 1}_{face}.pgm", "wb") as fh:
                    fh.write(b"P5\n%d %d\n255\n" % (S, S) + rel.tobytes())
                ce[face] = (rel.astype(np.float32) / 255.0)[None]
        frames.append(fr); flows.append(fl); certs.append(ce)
    return frames, flows, certs


def argv(d, ov, n, extra=()):
    return ["-input_pattern", f"{d}/in_%03d_%d.ppm", "-flow_pattern", f"{d}/bw_[%d]_{{%d}}_%d.flo",
            "-occlusions_pattern", f"{d}/rel_[%d]_{{%d}}_%d.pgm", "-output_prefix", f"{d}/out", "-overlap_pixel_w", str(ov),
            "-overlap_pixel_h", str(ov), "-num_frames", str(n), "-out_equi", "-out_cubemap", "-out_equi_w", "96",
            "-out_equi_h", "48", *extra]


def read_eval(path, nq):
    rows = open(path).read().strip().split("\n")
    assert len(rows) == 2 * nq, rows
    return [[float(v) for v in r.split(";")] for r in rows[:nq]], [float(r) for r in rows[nq:]]


S, OV, NF = 64, 20, 3
VARIANTS = {
    "plain": ((), {}),
    "no_consistency_eval": (("-no_consistency_eval",), dict(no_consistency_eval=True)),
    "backward_eval": (("-backward_eval",), dict(backward_eval=True)),
    "fix_occlusions_eval": (("-fix_occlusions_eval",), dict(fix_occlusions_eval=True)),
    "eval_patterns": (None, dict(invert_occlusions_eval=True)),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_vr_evaluate_vs_restatement(tmp_path, monkeypatch, variant):
    """3 VR frames x 6 faces with -evaluate and no loss network: the gradient, seam and temporal rows against the hook of the
    driver restatement, the perceptual rows nan, the averages over num_frames x 6; the stylized outputs are those of the run
    without -evaluate, bit for bit."""
    d = str(tmp_path)
    monkeypatch.chdir(tmp_path)  # no models/vgg16.t7 here: the perceptual terms are nan
    frames, flows, certs = write_clip(d, S, NF)
    extra, hook_kw = VARIANTS[variant]
    eval_flows = eval_certs = None
    if extra is None:  # separate evaluation flows and certainties, inverted
        _, eval_flows, eval_certs = write_clip(d, S, NF, prefix="ev_", seed0=5)
        extra = ("-flow_pattern_eval", f"{d}/ev_bw_[%d]_{{%d}}_%d.flo", "-occlusions_pattern_eval",
                 f"{d}/ev_rel_[%d]_{{%d}}_%d.pgm", "-invert_occlusions_eval")
    drv = vr.main(argv(d, OV, NF, ("-evaluate", "-evaluation_file", f"{d}/eval.txt") + tuple(extra)), model_vid=FakeGpuNet())
    ref = ve.EvalVRRef(S, S, OV, OV, 3, 96, 48)
    outs, table = ve.run_vr_clip_eval(ref, FakeRefNet(), frames, flows, certs, hook_kw=hook_kw, eval_flows=eval_flows,
                                      eval_certs=eval_certs)
    nq = 6 if variant == "no_consistency_eval" else 7
    rows, avgs = read_eval(f"{d}/eval.txt", nq)
    assert len(table) == nq and all(len(r) == 6 * NF for r in rows)
    for q in (0, 1, 2, 3):  # gradx, grady, gradmag, edge
        for k, (g, r) in enumerate(zip(rows[q], table[q])):
            assert same(g, float(r), GRAD_REL), (q, k, g, r)
    assert all(v == 0.0 for v in rows[3][0::6] + rows[3][5::6])  # modes 0 and 5 have no seam term
    assert all(v == 0.0 for q in (0, 1, 2) for v in rows[q][0::6])  # nor does mode 0 a gradient term
    assert all(math.isnan(v) for v in rows[4] + rows[5])
    if nq == 7:
        assert rows[6][:6] == [0.0] * 6 and all(t > 0 for t in rows[6][6:])
        for k, (g, r) in enumerate(zip(rows[6], table[6])):
            assert abs(g - r) <= 1e-9 + 1e-7 * r, (k, g, r)
    for q in range(nq):  # sum / opt.num_frames, which the driver has multiplied by 6
        want = sum(rows[q]) / (6 * NF)
        assert same(avgs[q], want, 1e-12), (q, avgs[q], want)
    # the same clip without -evaluate: outputs and the re-blended faces bit-identical
    plain = vr.main(argv(d, OV, NF), model_vid=FakeGpuNet())
    for k in range(1, NF + 1):
        for key in ("equi", "cubemap"):
            assert torch.equal(drv.outputs[k][key], plain.outputs[k][key]), (k, key)
            assert np.array_equal(drv.outputs[k][key].cpu().numpy(), outs[k - 1][key]), (k, key)
    for face in range(1, 7):
        assert torch.equal(drv.prev_last_segments[face], plain.prev_last_segments[face]), face
        assert torch.equal(drv.last_segments[face], plain.last_segments[face]), face


def test_vr_evaluate_with_loss_network(tmp_path, monkeypatch):
    """A seeded VGG-16 .t7 and a style image already at -style_image_size: rows 5 and 6 hold, per face, the content and the
    style loss of the loaded face against its stylized face (swapped as func_eval's `style_loss, content_loss =` reads them)."""
    from PIL import Image

    d = str(tmp_path)
    monkeypatch.chdir(tmp_path)
    n = 2
    frames, flows, certs = write_clip(d, S, n)
    mods = percep.vgg16_modules(8)
    t7.write_loss_network(f"{d}/vgg16.t7", mods)
    yy, xx = np.mgrid[0:70, 0:90]
    style = np.stack([0.5 + 0.5 * np.sin(xx / 3.0 + c) * np.cos(yy / 5.0 - c) for c in range(3)]).astype(np.float32)
    synth.write_ppm(f"{d}/style.ppm", style)
    stylized = []
    orig = vr.VRDriver.func_save_image

    def record(self, opt, i, frame, dtype=None):
        stylized.append(frame.detach().cpu().numpy().copy())
        return orig(self, opt, i, frame, dtype)

    monkeypatch.setattr(vr.VRDriver, "func_save_image", record)
    base = argv(d, OV, n, ("-evaluate", "-loss_network", f"{d}/vgg16.t7", "-style_image", f"{d}/style.ppm",
                           "-style_image_size", "90", "-style_weights", "1,2,3,4", "-content_weights", "5"))
    vr.main(base + ["-evaluation_file", f"{d}/eval.txt"], model_vid=FakeGpuNet())
    rows, avgs = read_eval(f"{d}/eval.txt", 7)
    ora = percep_oracle.PercepOracle(mods, [16], [5.0], [4, 9, 16, 23], [1.0, 2.0, 3.0, 4.0])
    ora.set_style_target(np.asarray(Image.open(f"{d}/style.ppm"), np.float32).transpose(2, 0, 1) / 255.0)
    assert len(stylized) == 6 * n and len(rows[4]) == len(rows[5]) == 6 * n
    worst = 0.0
    for i in range(1, 6 * n + 1):
        mode, f = (i - 1) % 6, (i - 1) // 6
        rc, rs = ora.evaluate(frames[f][vr_oracle.PROC_ORDER[mode]], stylized[i - 1])[:2]
        assert abs(rows[4][i - 1] - rc) <= LOSS_BAR * rc, (i, rows[4][i - 1], rc)
        assert abs(rows[5][i - 1] - rs) <= LOSS_BAR * rs, (i, rows[5][i - 1], rs)
        worst = max(worst, abs(rows[4][i - 1] - rc) / rc, abs(rows[5][i - 1] - rs) / rs)
    print(f"\nVR -evaluate perceptual rows: worst relative error {worst:.2e}")
    assert all(math.isfinite(v) for q in range(7) for v in rows[q])
    with pytest.raises(_lib.FavError) as e:
        vr.main(argv(d, OV, n, ("-evaluate", "-loss_network", f"{d}/missing.t7")), model_vid=FakeGpuNet())
    assert e.value.status == _lib.FAV_ERR_IO
