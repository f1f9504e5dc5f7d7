"""fast_artistic_video.lua -- the plain-video driver: CLI flags (:21-67), filename patterns (:70-77), callbacks
(:93-172) and main (:174-189).  `python -m fav_b200.video -input_pattern frame_%04d.ppm -flow_pattern ... `.

File formats: frames PPM/PNG/JPG (PIL), certainty PGM (the consistencyChecker output), flow Middlebury .flo.
PNG quantisation of image.save lives in the un-vendored torch `image` rock (unpinned): clamp to [0,1], x255, round.
"""
from __future__ import annotations

import argparse
import os
import re
import sys

import numpy as np
import torch

from . import _lib, consistencyChecker, core, flowFileLoader, utils


def build_parser():
    p = argparse.ArgumentParser(prefix_chars="-", description="Stylize a video with a trained feedforward model")
    a = p.add_argument
    a("-model_img", default="self"); a("-model_vid", default="synthetic:candy")
    a("-num_frames", type=int, default=9999); a("-continue_with", type=int, default=1)
    a("-input_pattern", default=""); a("-output_prefix", default="out")
    a("-flow_pattern", default=""); a("-occlusions_pattern", default="")
    # forward flows, e.g. forward_{%d}_[%d].flo: with an empty -occlusions_pattern the certainty of frame i is computed on the GPU
    # from backward_i_{i-1}, forward_{i-1}_i and frame i, as makeOptFlow_deepflow.sh:58-60 computes reliable_i_{i-1}.pgm
    a("-flow_pattern_forward", default="")
    a("-invert_occlusion", action="store_true"); a("-occlusions_min_filter", type=int, default=7)
    a("-fill_occlusions", default="vgg-mean"); a("-fix_occlusions", action="store_true")
    a("-median_filter", type=int, default=3)  # declared but unused by the plain driver (fast_artistic_video.lua:39)
    a("-scale_factor", type=float, default=1); a("-backward", action="store_true")
    a("-create_inconsistent", action="store_true")
    a("-gpu", type=int, default=0); a("-backend", default="cuda"); a("-use_cudnn", type=int, default=1)
    a("-cudnn_benchmark", type=int, default=0); a("-evaluate", action="store_true")
    a("-evaluation_file", default="evaluation.txt"); a("-flow_pattern_eval", default=""); a("-occlusions_pattern_eval", default="")
    a("-invert_occlusion_eval", action="store_true"); a("-fix_occlusions_eval", action="store_true"); a("-backward_eval", action="store_true")
    a("-model_img_arch", default="")
    # the perceptual terms of -evaluate (fast_artistic_video.lua:57-67); no -loss_network and no models/vgg16.t7: reported as nan
    a("-content_weights", default="1.0"); a("-content_layers", default="16")
    a("-loss_network", default=None); a("-style_image", default="images/styles/candy.jpg"); a("-style_image_size", type=int, default=256)
    a("-style_weights", default="1.0"); a("-style_layers", default="4,9,16,23"); a("-style_target_type", default="gram", choices=["gram", "mean"])
    a("-pipeline", type=int, default=1)  # 1: threaded decode / encode around the host-buffer session (f-2); 0: synchronous driver
    a("-arch", default=core.synth.DEFAULT_ARCH)
    # not a reference option: "fp16" runs every convolution of the nets in one fp16 pass (fav_net_set_precision)
    a("-precision", default="pair", choices=["pair", "fp16"])
    return p


def getFormatedFlowFileName(pattern: str, fromIndex: int, toIndex: int) -> str:
    """fast_artistic_video.lua:70-77: {fmt} is formatted with the from-index, [fmt] with the to-index."""
    s = re.sub(r"\{(.*?)\}", lambda m: m.group(1) % fromIndex, pattern)
    return re.sub(r"\[(.*?)\]", lambda m: m.group(1) % toIndex, s)


def load_image(path: str, channels: int) -> torch.Tensor:
    """image.load(path, channels): float [0,1], CxHxW.  Binary PPM / PGM files (what the reference's pipelines produce,
    run-deepflow.sh / makeOptFlow.sh) go through the native reader (byte / 255 in fp32, as image.load); anything else
    through PIL."""
    if path.lower().endswith((".ppm", ".pgm", ".pnm")):
        import ctypes as C

        w_, h_, c_ = C.c_int(), C.c_int(), C.c_int()
        if _lib.lib.fav_pnm_read_header(path.encode(), C.byref(w_), C.byref(h_), C.byref(c_)) == _lib.FAV_OK and c_.value == channels:
            out = np.empty((channels, h_.value, w_.value), np.float32)
            _lib.check(_lib.lib.fav_pnm_read_f32(path.encode(), out.ctypes.data_as(C.c_void_p), out.size, C.c_float(255.0)))
            return torch.from_numpy(out)
    from PIL import Image

    im = Image.open(path).convert("RGB" if channels == 3 else "L")
    a = np.asarray(im, dtype=np.float32) / 255.0
    return torch.from_numpy(a.transpose(2, 0, 1).copy() if channels == 3 else a[None].copy())


_SAVE_POOL = None
_SAVE_PENDING = []


def save_image(path: str, img: torch.Tensor, background: bool = False) -> None:
    """image.save(path, img): clamp to [0,1], x255, round -> 8-bit PNG.  Quantised on the tensor's device, encoded by the
    native writer (fav_png_write: Sub filter, zlib level 1 + Z_RLE, concurrent deflate bands -- the cube-map strips of the VR
    driver are 12288 x 2048).  background=True returns after the device->host copy and encodes on a worker thread
    (flush_saves() waits); the pixels any PNG decoder returns are the same either way."""
    import ctypes as C

    a = (img.detach().clamp(0, 1) * 255.0 + 0.5).floor().clamp(0, 255).byte()
    if a.dim() == 2:
        a = a[None]
    a = a.permute(1, 2, 0).contiguous().cpu().numpy()
    H, W, Cn = a.shape
    if Cn not in (1, 3):
        raise _lib.FavError(_lib.FAV_ERR_INVALID, f"save_image: {Cn} channels")
    nthreads = max(1, min(16, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)))

    def write():
        _lib.check(_lib.lib.fav_png_write(path.encode(), a.ctypes.data_as(C.c_void_p), W, H, Cn, 1, nthreads))

    if not background:
        write()
        return
    global _SAVE_POOL
    if _SAVE_POOL is None:
        from concurrent.futures import ThreadPoolExecutor

        _SAVE_POOL = ThreadPoolExecutor(max_workers=3)
    _SAVE_PENDING.append(_SAVE_POOL.submit(write))


def flush_saves() -> None:
    """Wait for the background PNG writes (and surface their errors)."""
    while _SAVE_PENDING:
        _SAVE_PENDING.pop(0).result()


class Driver:
    def __init__(self, opt):
        self.opt = opt
        self.last_frame_stylized = None  # fast_artistic_video.lua:89
        self.prev_last_frame_stylized = None
        self.last_frame = None

    def func_load_image(self, opt, i, dtype):  # :93-97
        path = opt.input_pattern % i
        if not utils.file_exists(path):
            return None
        self.last_frame = load_image(path, 3)
        return self.last_frame

    def fix_occlusions(self, flow, occluded):  # :79-86
        tmp = utils.warp_image(torch.ones_like(occluded), flow)
        occluded.mul_(((tmp - 0.5).sign()).clamp(min=0))

    def func_load_cert(self, opt, i, dtype):  # :99-112
        flowFileName = getFormatedFlowFileName(opt.flow_pattern, i - 1, i)
        if opt.flow_pattern_forward:  # the checker's 4-argument mode on frame i (loaded just before by func_load_image)
            fwFileName = getFormatedFlowFileName(opt.flow_pattern_forward, i - 1, i)
            utils.wait_for_file(fwFileName)
            utils.wait_for_file(flowFileName)
            bw = torch.from_numpy(flowFileLoader.load(flowFileName, layout=1)).cuda()
            fw = torch.from_numpy(flowFileLoader.load(fwFileName, layout=1)).cuda()
            cert = consistencyChecker.check(bw, fw, self.last_frame.cuda() * 255.0, want_cert=True)[1][None]
        else:
            certFileName = getFormatedFlowFileName(opt.occlusions_pattern, i - 1, i)
            utils.wait_for_file(certFileName)
            cert = load_image(certFileName, 1).cuda()
        if opt.invert_occlusion:
            cert = 1.0 - cert
        if opt.fix_occlusions:
            flow = torch.from_numpy(flowFileLoader.load(flowFileName)).cuda()
            self.fix_occlusions(flow, cert)
        return cert

    def func_make_last_frame_warped(self, opt, i, dtype, cert_mask=None):  # :153-158
        flowFileName = getFormatedFlowFileName(opt.flow_pattern, i - 1, i)
        flow = torch.from_numpy(flowFileLoader.load(flowFileName)).cuda()
        return core.FusedWarp(self.last_frame_stylized, flow), None

    def func_load_flow_cert_eval(self, opt, i, dtype):  # :114-126
        flow = torch.from_numpy(flowFileLoader.load(getFormatedFlowFileName(opt.flow_pattern_eval, i - 1, i))).cuda()
        cert = load_image(getFormatedFlowFileName(opt.occlusions_pattern_eval, i - 1, i), 1).cuda()
        if opt.invert_occlusion_eval:
            cert = 1.0 - cert
        if opt.fix_occlusions_eval:
            self.fix_occlusions(flow, cert)
        return flow, cert

    def func_eval(self, opt, i, func_percept_loss, dtype):  # :128-151
        # :129 unpacks evaluate_image's (content, style) pair as `style_loss, content_loss`, so the first row of the evaluation
        # file holds the content losses and the second the style losses; reproduced as written.  Without a loss network
        # (core.make_evaluate_image returns None) both are nan.
        nan = float("nan")
        style_loss, content_loss = func_percept_loss(self.last_frame, self.last_frame_stylized) if func_percept_loss else (nan, nan)
        if i > 1:
            flow_eval, cert_eval = self.func_load_flow_cert_eval(opt, i, dtype)
            if opt.backward_eval:
                t = utils.temporal_loss(self.last_frame_stylized, self.prev_last_frame_stylized, flow_eval, cert_eval)
            else:
                t = utils.temporal_loss(self.prev_last_frame_stylized, self.last_frame_stylized, flow_eval, cert_eval)
            return [style_loss, content_loss, t], 3
        return [style_loss, content_loss, 0.0], 3

    def func_save_image(self, opt, i, img, dtype=None):  # :160-170
        out_path = "%s-%05d.png" % (opt.output_prefix, i)
        print("Writing output image to " + out_path)
        d = os.path.dirname(out_path)
        if d and not os.path.isdir(d):
            os.makedirs(d)
        save_image(out_path, img)
        self.prev_last_frame_stylized = self.last_frame_stylized
        self.last_frame_stylized = img.clone()  # fp32, unclamped: NOT the PNG

    @staticmethod
    def func_is_single_image(i, opt):  # :172
        return i == 1 or opt.create_inconsistent


# ---------------------------------------------------------------------------------------------------------------------
# f-2: the same driver as a PIPELINE on the host-buffer session (fav_session_*): decode threads fill pinned ring buffers
# (frame PPM/PNG -> fp32 planes, .flo -> (dy,dx) planes, certainty PGM), the main thread only enqueues frames
# (3 CUDA streams inside the session: H2D / compute / D2H), encoder threads wait for ONE frame each (fav_session_frame_done)
# and write its PNG.  Filename patterns ([%d] / {%d}) and the wait-for-file protocol of the flow / occlusion producers
# (utils.lua:74-80) are those of the synchronous driver; the PNGs are bit-identical to it (tests/test_gpu_net.py).
# The reference decodes, uploads, computes, downloads and encodes strictly one after the other
# (fast_artistic_video.lua:93-170); at H100 speeds that host work, not the GPU, bounds the frame rate.
# ---------------------------------------------------------------------------------------------------------------------
def _read_planes(path: str, channels: int, out: torch.Tensor) -> None:
    """image.load(path, channels) into a preallocated (pinned) [C,H,W] tensor."""
    if path.lower().endswith((".ppm", ".pgm", ".pnm")):
        import ctypes as C

        _lib.check(_lib.lib.fav_pnm_read_f32(path.encode(), C.c_void_p(out.data_ptr()), out.numel(), C.c_float(255.0)))
    else:
        out.copy_(load_image(path, channels))


def _png_bytes(img: torch.Tensor) -> np.ndarray:
    """the quantisation of save_image on a host tensor (same fp32 operations)"""
    a = img.numpy()
    return np.clip(np.floor(np.clip(a, 0.0, 1.0) * np.float32(255.0) + np.float32(0.5)), 0, 255).astype(np.uint8).transpose(1, 2, 0)


def pipeline_eligible(opt) -> bool:
    return not (opt.backward or opt.evaluate or opt.fix_occlusions or opt.create_inconsistent or opt.fill_occlusions != "vgg-mean"
                or float(opt.scale_factor) != 1 or opt.continue_with != 1)


def _native_ok(opt) -> bool:
    """the native pipeline decodes binary PPM / PGM only (what the reference's scripts extract with ffmpeg,
    stylizeVideo_*.sh: frame_%04d.ppm, and what consistencyChecker writes)"""
    return opt.input_pattern.lower().endswith(".ppm") and (opt.flow_pattern_forward != ""
                                                           or opt.occlusions_pattern.lower().endswith(".pgm"))


def run_native(opt, model_vid=None, model_img=None, n_decode=None, n_encode=None, depth=None, png_level=1):
    """f-2 in C++ (csrc/video_pipeline.cu): decoder / encoder std::threads around the host-buffer session."""
    import ctypes as C

    from . import session

    first = opt.input_pattern % 1
    if not utils.file_exists(first):
        return dict(frames=0, seconds=0.0)
    w_, h_, c_ = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib.fav_pnm_read_header(first.encode(), C.byref(w_), C.byref(h_), C.byref(c_)))
    H, W = h_.value, w_.value
    torch.cuda.set_device(max(0, int(opt.gpu)))
    model = model_vid if model_vid is not None else core.load_model(opt.model_vid, opt.arch)
    if model_img is None and opt.model_img not in ("self", "", None):
        model_img = core.load_model(opt.model_img, opt.model_img_arch or opt.arch, in_dim=3)
    core.set_precision(opt, model, model_img)
    sess = session.Session(model, H, W)
    if model_img is not None:
        sess.set_image_model(model_img)
    d = os.path.dirname(opt.output_prefix)
    if d and not os.path.isdir(d):
        os.makedirs(d)
    cpus = os.cpu_count() or 8
    n_decode = n_decode or max(2, min(16, cpus // 8))
    n_encode = n_encode or max(4, min(64, cpus // 2))
    depth = depth or (n_decode + n_encode + 4)
    nfr, secs = C.c_int(), C.c_double()
    if opt.flow_pattern_forward:
        _lib.check(_lib.lib.fav_video_pipeline_run_flows(sess._h, H, W, opt.input_pattern.encode(), opt.flow_pattern.encode(),
                                                         opt.flow_pattern_forward.encode(), opt.output_prefix.encode(),
                                                         int(opt.num_frames), int(opt.occlusions_min_filter), n_decode, n_encode,
                                                         depth, png_level, C.byref(nfr), C.byref(secs)))
    else:
        _lib.check(_lib.lib.fav_video_pipeline_run(sess._h, H, W, opt.input_pattern.encode(), opt.flow_pattern.encode(),
                                                   opt.occlusions_pattern.encode(), opt.output_prefix.encode(), int(opt.num_frames),
                                                   int(opt.occlusions_min_filter), 1 if opt.invert_occlusion else 0, n_decode,
                                                   n_encode, depth, png_level, C.byref(nfr), C.byref(secs)))
    if nfr.value:
        print("Stylized %d frames in %.3f s (%.1f frames/s, files -> PNG, native pipeline)" % (nfr.value, secs.value, nfr.value / secs.value))
    return dict(frames=nfr.value, seconds=secs.value)


def run_pipelined(opt, depth: int = 8, n_decode: int = 6, n_encode: int = 12, model_vid=None, model_img=None):
    import time
    from concurrent.futures import ThreadPoolExecutor
    from PIL import Image

    from . import session

    n = 0
    while n < opt.num_frames and utils.file_exists(opt.input_pattern % (n + 1)):  # func_load_image returns nil -> stop (:93-97)
        n += 1
    if n == 0:
        return dict(frames=0, seconds=0.0)
    first = load_image(opt.input_pattern % 1, 3)
    H, W = first.shape[-2:]
    dev = torch.device("cuda", max(0, int(opt.gpu)))
    torch.cuda.set_device(dev)
    model = model_vid if model_vid is not None else core.load_model(opt.model_vid, opt.arch)
    if model_img is None and opt.model_img not in ("self", "", None):
        model_img = core.load_model(opt.model_img, opt.model_img_arch or opt.arch, in_dim=3)
    core.set_precision(opt, model, model_img)
    sess = session.Session(model, H, W)
    if model_img is not None:
        sess.set_image_model(model_img)
    pin = lambda *shape: torch.empty(shape, dtype=torch.float32).pin_memory()
    slots = [dict(content=pin(3, H, W), flow=pin(2, H, W), cert=pin(1, H, W), out=pin(3, H, W)) for _ in range(depth)]
    d = os.path.dirname(opt.output_prefix)
    if d and not os.path.isdir(d):
        os.makedirs(d)

    def decode(i, slot):  # i is the 1-based frame index
        _read_planes(opt.input_pattern % i, 3, slot["content"])
        if i > 1:
            flowFileName = getFormatedFlowFileName(opt.flow_pattern, i - 1, i)
            certFileName = getFormatedFlowFileName(opt.occlusions_pattern, i - 1, i)
            utils.wait_for_file(certFileName)  # func_load_cert :101-102
            _read_planes(certFileName, 1, slot["cert"])
            if opt.invert_occlusion:
                slot["cert"].mul_(-1.0).add_(1.0)
            utils.wait_for_file(flowFileName)
            flowFileLoader.load(flowFileName, out=slot["flow"].numpy())
        return slot

    def encode(i, k, slot):
        sess.frame_done(k)  # this frame's D2H only; later frames keep flowing
        out_path = "%s-%05d.png" % (opt.output_prefix, i)
        Image.fromarray(_png_bytes(slot["out"])).save(out_path)
        return slot

    t0 = time.perf_counter()
    free = list(slots)
    with ThreadPoolExecutor(n_decode) as dpool, ThreadPoolExecutor(n_encode) as epool:
        dec, enc = {}, []
        nxt = 1
        for i in range(1, n + 1):
            while nxt <= n and free:  # keep the decoders `depth` frames ahead
                dec[nxt] = dpool.submit(decode, nxt, free.pop())
                nxt += 1
            if i not in dec:  # every slot is in flight: wait for the oldest encoder to give one back
                free.append(enc.pop(0).result())
                dec[i] = dpool.submit(decode, i, free.pop())
                nxt = max(nxt, i + 1)
            slot = dec.pop(i).result()
            if i == 1:
                sess.run_image(slot["content"], slot["out"])
            else:
                sess.run_next_image(slot["content"], slot["flow"], slot["cert"][0], slot["out"], opt.occlusions_min_filter)
            enc.append(epool.submit(encode, i, i - 1, slot))
            while enc and enc[0].done():
                free.append(enc.pop(0).result())
        for f in enc:
            f.result()
    sess.sync()
    dt = time.perf_counter() - t0
    print("Stylized %d frames in %.3f s (%.1f frames/s, files -> PNG, pipelined)" % (n, dt, n / dt))
    return dict(frames=n, seconds=dt)


def main(argv=None):
    opt = build_parser().parse_args(argv)
    if opt.input_pattern == "":
        raise SystemExit("Must give -input_pattern")  # :177-179
    if opt.flow_pattern_forward:  # certainties computed from the flow pair and the frame (4-argument checker)
        if opt.flow_pattern == "":
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "-flow_pattern_forward needs -flow_pattern (the backward flows)")
        if opt.occlusions_pattern != "":
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "give either -occlusions_pattern or -flow_pattern_forward")
        if opt.invert_occlusion:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "-invert_occlusion inverts loaded PGMs; the computed certainty is not inverted")
    elif not opt.create_inconsistent and (opt.flow_pattern == "" or opt.occlusions_pattern == ""):
        raise SystemExit("Must give -flow_pattern and -occlusions_pattern")  # :180-182
    if opt.pipeline and pipeline_eligible(opt):
        if _native_ok(opt):
            return run_native(opt)
        if not opt.flow_pattern_forward:  # the Python pipeline reads certainty PGMs; computed ones take the driver below
            return run_pipelined(opt)
    d = Driver(opt)
    core.run_fast_neural_video(opt, d.func_load_image, d.func_load_cert, d.func_eval, d.func_make_last_frame_warped,
                               d.func_is_single_image, d.func_save_image)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main(sys.argv[1:])
