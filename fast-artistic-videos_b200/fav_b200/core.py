"""fast_artistic_video_core.lua -- `run_fast_neural_video(opt, func_load_image, func_load_cert, func_eval,
func_make_last_frame_warped, func_is_single_image, func_save_image)` (:34) with the same callback protocol.

Differences that are design, not semantics:
  * the ~10 elementwise kernels + 2 torch.cat copies of run_next_image (:166-171) are ONE fused kernel
    (fav_temporal_input / fav_run_next_image);
  * `func_make_last_frame_warped` may return a `FusedWarp(prev, flow)` request instead of an already warped image;
    the warp then happens inside that fused kernel.  A plain tensor (the reference protocol, e.g. the VR driver's
    blended prior) is still accepted: it is fed through the same kernel with a zero flow, which is exact
    (weights 1,0,0,0);
  * `generate_fill` (:108-117) draws torch.rand even when the result is discarded ('vgg-mean'); here nothing is drawn
    for 'vgg-mean' and 'uniform-random' draws on the GPU (the reference RNG stream is not reproducible anyway).
-evaluate (:76-98,214-239): the temporal loss is computed (utils.temporal_loss, one fused kernel); the content and style losses
run through the loss network on the GPU (fav_b200/percep.py) when -loss_network names one or models/vgg16.t7 exists, and are
reported as NaN otherwise.
"""
from __future__ import annotations

import time
from dataclasses import dataclass

import torch

from . import _lib, models_video, synth, utils


@dataclass
class FusedWarp:
    """Deferred utils.warp_image(prev, flow): executed inside the fused temporal-input kernel."""
    prev: torch.Tensor  # 3xHxW RGB, unclamped fp32 (last_frame_stylized, fast_artistic_video.lua:169)
    flow: torch.Tensor  # 2xHxW (dy, dx)
    border_mode: int = _lib.BORDER_PER_TAP


def _opt(opt, k, d=None):
    return opt.get(k, d) if isinstance(opt, dict) else getattr(opt, k, d)


def set_precision(opt, *models) -> None:
    """-precision pair|fp16 (an addition, StyleNet.set_precision) on every net the driver runs: the video model and the image
    model, whichever driver (native pipeline, session, synchronous loop) then runs them."""
    mode = _opt(opt, "precision", "pair")
    for m in models:
        if m is not None and getattr(m, "precision", "pair") != mode:
            m.set_precision(mode)


def load_model(path_or_style: str, arch: str = synth.DEFAULT_ARCH, in_dim: int = 7) -> models_video.StyleNet:
    """get_model (core.lua:38-57): a Torch7 `.t7` checkpoint (fav_b200/t7.py; the arch is recovered from the module
    tree), a `.npz` state dict, or `synthetic:<style>` = seeded random-init weights (no network here to fetch the
    released checkpoints)."""
    if path_or_style.endswith(".npz"):
        import numpy as np

        w = dict(np.load(path_or_style))
        norm = "batch" if any(k.endswith(".running_var") for k in w) else "instance"
        return models_video.StyleNet(arch, in_dim=in_dim, norm=norm).load_state(w)
    if path_or_style.endswith(".t7"):  # torch.load(path).model (core.lua:39-47)
        from . import t7

        geo = {}
        try:
            t7_arch, state, tanh_c, pad = t7.load_checkpoint(path_or_style, geo)
        except t7.GeometryError as e:  # a padding_type / module layout this implementation does not run
            raise _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, str(e)) from None
        cin = int(next(v for k, v in state.items() if k == "l0.weight").shape[1])
        net = models_video.StyleNet(t7_arch, geo["padding_type"], tanh_constant=tanh_c, in_dim=cin, norm=geo["norm"])
        want = synth.reflect_start_pad(synth.parse_arch(t7_arch, cin), geo["padding_type"])
        if pad != want:  # the file's SpatialReflectionPadding must be the one the arch implies (train_video.lua:319-324)
            raise _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, f"{path_or_style}: SpatialReflectionPadding({pad}) in the checkpoint, "
                                f"the arch '{t7_arch}' with padding_type {geo['padding_type']} implies {want}")
        return net.load_state(state)
    style = path_or_style.split(":", 1)[-1]
    return models_video.synthetic_model(style, arch, in_dim)


def make_evaluate_image(opt):
    """The perceptual-loss set-up of core.lua:74-98 and evaluate_image (:101-106), or None when no loss network is available
    (-loss_network not given and no models/vgg16.t7).  A -loss_network or -style_image that was named and is missing is an
    I/O error."""
    import os

    from . import percep

    path = _opt(opt, "loss_network", None)
    if path in (None, ""):
        path = os.path.join("models", "vgg16.t7")
        if not os.path.exists(path):
            return None
    elif not os.path.exists(path):
        raise _lib.FavError(_lib.FAV_ERR_IO, f"-loss_network {path}: no such file")
    content_layers, content_weights = percep.parse_layers(_opt(opt, "content_layers", "16"), _opt(opt, "content_weights", "1.0"))
    style_layers, style_weights = percep.parse_layers(_opt(opt, "style_layers", "4,9,16,23"), _opt(opt, "style_weights", "1.0"))
    crit = percep.PerceptualCriterion.from_t7(path, content_layers, content_weights, style_layers, style_weights,
                                              _opt(opt, "style_target_type", "gram"))
    style_path = _opt(opt, "style_image", "images/styles/candy.jpg")
    if not os.path.exists(style_path):
        raise _lib.FavError(_lib.FAV_ERR_IO, f"-style_image {style_path}: no such file")
    from .video import load_image  # image.load(opt.style_image, 3, 'float')

    style = percep.scale_style_image(load_image(style_path, 3), int(_opt(opt, "style_image_size", 256)))
    crit.set_style_target(style.cuda())

    def evaluate_image(content_img, stylized_img):
        return crit.evaluate(content_img, stylized_img)

    evaluate_image.criterion = crit
    return evaluate_image


def run_fast_neural_video(opt, func_load_image, func_load_cert, func_eval, func_make_last_frame_warped,
                          func_is_single_image, func_save_image, model_vid=None, model_img=None):
    dtype = "torch.CudaTensor"  # utils.setup_gpu (utils.lua:43-66): this implementation is GPU-only
    dev = torch.device("cuda", int(_opt(opt, "gpu", 0)) if int(_opt(opt, "gpu", 0)) >= 0 else 0)
    torch.cuda.set_device(dev)
    evaluate = bool(_opt(opt, "evaluate", False))  # :76-98,214-239 -- see the evaluation block at the end of the loop
    scale_factor = float(_opt(opt, "scale_factor", 1))
    model = model_vid if model_vid is not None else load_model(_opt(opt, "model_vid"), _opt(opt, "arch", synth.DEFAULT_ARCH))
    # get_model (core.lua:59-69): 'self' -> model_img = nil, the video model also stylizes single images
    model_img = model_img if model_img is not None else (
        None if _opt(opt, "model_img", "self") in ("self", "", None)
        else load_model(_opt(opt, "model_img"), _opt(opt, "arch_img", _opt(opt, "arch", synth.DEFAULT_ARCH)), in_dim=3))
    set_precision(opt, model, model_img)
    evaluate_image = make_evaluate_image(opt) if evaluate else None
    fill_mode = _opt(opt, "fill_occlusions", "vgg-mean")
    assert fill_mode in ("vgg-mean", "uniform-random")

    def generate_fill(H, W, cert):  # core.lua:108-117
        if fill_mode == "vgg-mean":
            return None
        from . import preprocess

        rnd = preprocess.vgg.preprocess(torch.rand((1, 3, H, W), device=dev))[0]
        return rnd * (1.0 - cert)

    def run_image(img):  # core.lua:121-158
        t1 = time.perf_counter()
        H, W = img.shape[-2:]
        if model_img is not None:  # core.lua:146: model_img:forward(img_pre), between the two image.scale calls of :127-152
            out = model_img.run_image(img.to(dev), scale_factor=scale_factor)
        elif scale_factor != 1:  # core.lua:135: the fill has the unscaled size, so torch.cat fails
            raise _lib.FavError(_lib.FAV_ERR_INVALID, f"-scale_factor {scale_factor} needs -model_img: the video model's input "
                                "would join the scaled frame with an unscaled fill (fast_artistic_video_core.lua:133-138)")
        else:
            out = model.run_image(img.to(dev), generate_fill(H, W, torch.zeros((1, H, W), device=dev)))
        print("Elapsed time for stylizing frame independently:%f" % (time.perf_counter() - t1))
        return out

    def run_next_image(H, W, new_content_img, cert_mask, i):  # core.lua:161-180
        res = func_make_last_frame_warped(opt, i, dtype, cert_mask)
        prior, flow_mask = res if isinstance(res, tuple) else (res, None)
        t1 = time.perf_counter()
        cert = cert_mask.reshape(H, W)
        fill = generate_fill(H, W, cert[None])
        if isinstance(prior, FusedWarp):
            out = model.run_next_image(new_content_img.to(dev), prior.prev, prior.flow, cert, fill,
                                       None if flow_mask is None else flow_mask.reshape(H, W), prior.border_mode)
        else:  # already warped by the callback: identity flow keeps the values bit-exact
            zero = torch.zeros((2, H, W), device=dev)
            out = model.run_next_image(new_content_img.to(dev), prior.to(dev).reshape(3, H, W), zero, cert, fill,
                                       None if flow_mask is None else flow_mask.reshape(H, W))
        print("Elapsed time for stylizing frame:%f" % (time.perf_counter() - t1))
        return out

    eval_tabl, eval_sum = [], []
    backward = bool(_opt(opt, "backward", False))
    num_frames = int(_opt(opt, "num_frames", 9999))
    start_idx = num_frames - 1 if backward else int(_opt(opt, "continue_with", 1))  # :189-191
    end_idx = 1 if backward else num_frames
    inc = -1 if backward else 1
    i = start_idx
    while (i >= end_idx) if backward else (i <= end_idx):  # :194
        img = func_load_image(opt, i, dtype)
        if img is None:
            break
        H, W = img.shape[-2:]
        if func_is_single_image(i, opt):
            nxt = run_image(img)
        else:
            cert = func_load_cert(opt, i, dtype)
            r = int(_opt(opt, "occlusions_min_filter", 7))
            cert = utils.min_filter(cert.to(dev).reshape(1, H, W), r) if r > 1 else cert.to(dev)  # :207
            nxt = run_next_image(H, W, img, cert.reshape(1, 1, H, W), i)
        func_save_image(opt, i, nxt, dtype)
        if evaluate:
            # core.lua:214-226: func_eval -> { style_loss, content_loss, temporal_loss }; evaluate_image is None without a
            # loss network (the perceptual terms are then NaN); the temporal term is one fused warp + mask + MSE kernel.
            numbers, n_num = func_eval(opt, i, evaluate_image, dtype)
            for j in range(n_num):
                if j >= len(eval_tabl):
                    eval_tabl.append([]); eval_sum.append(0.0)
                eval_tabl[j].append(numbers[j]); eval_sum[j] += numbers[j]
        i += inc
    if evaluate:  # :231-240: one ';'-joined line per quantity, then the per-frame averages (sum / opt.num_frames)
        with open(_opt(opt, "evaluation_file", "evaluation.txt"), "a") as fh:
            for row in eval_tabl:
                fh.write(";".join(repr(float(v)) for v in row) + "\n")
            for t in eval_sum:
                fh.write(repr(float(t) / num_frames) + "\n")
        print("File written")
