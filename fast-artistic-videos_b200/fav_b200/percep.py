"""nn.PerceptualCriterion (fast_artistic_video/PerceptualCriterion.lua:27-155) for -evaluate: the content and style losses of a
stylized frame through a VGG-style loss network, computed by libfav_b200 (csrc/percep.cu) on the GPU.

Set-up as fast_artistic_video_core.lua:74-98: utils.parse_layers for the layer / weight strings, torch.load of the loss network
(fav_b200/t7.py), a loss layer after every named top-level module, the network trimmed after the deepest one, and the style
target captured from the style image scaled to -style_image_size.  evaluate() is evaluate_image (core.lua:101-106): it returns
(total_content_loss, total_style_loss).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib

AGG_TYPES = {"gram": 0, "mean": 1}


def parse_num_list(s: str) -> List[float]:
    """utils.parse_num_list (fast_artistic_video/utils.lua:9-17): comma-separated numbers."""
    return [float(v) for v in str(s).split(",")]


def parse_layers(layers_string: str, weights_string: str) -> Tuple[List[str], List[float]]:
    """utils.parse_layers (fast_artistic_video/utils.lua:20-40): comma-separated layer strings; a single weight is repeated for
    every layer, any other count mismatch is an error."""
    layers = str(layers_string).split(",")
    weights = parse_num_list(weights_string)
    if len(weights) == 1 and len(layers) > 1:
        weights = weights * len(layers)
    elif len(weights) != len(layers):
        raise ValueError(f'size mismatch between layers "{layers_string}" and weights "{weights_string}"')
    return layers, weights


def layer_index(layer_string: str) -> int:
    """A top-level layer string ('16') -> 16.  Nested strings ('2-1', layer_utils.lua:40-46) address modules inside containers;
    the loss networks this implementation runs are flat, so they are refused."""
    s = str(layer_string).strip()
    if "-" in s:
        raise _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, f"loss layer '{s}': nested layer strings are not supported (flat loss networks only)")
    return int(s)


# VGG-16 as loadcaffe converts it (the module list of models/vgg16.t7 up to pool5): conv3x3/pad 1 + ReLU, 2x2/2 max-poolings.
# Module indices: relu1_2 = 4, relu2_2 = 9, relu3_3 = 16, relu4_3 = 23 (the default -style_layers).
VGG16_CHANNELS = [[64, 64], [128, 128], [256, 256, 256], [512, 512, 512], [512, 512, 512]]


def vgg16_modules(seed: int = 0, ceil_mode: bool = False, scale: float = 1.0) -> List[dict]:
    """VGG-16's feature layers with seeded weights (He-normal, so activations keep their scale through the ReLUs; `scale`
    multiplies the first convolution).  There is no network here to fetch the released weights; the shapes are the real ones."""
    rng = np.random.default_rng(seed)
    mods, cin = [], 3
    for bi, block in enumerate(VGG16_CHANNELS):
        for cout in block:
            std = np.sqrt(2.0 / (cin * 9))
            w = (rng.standard_normal((cout, cin, 3, 3)) * std).astype(np.float32)
            if cin == 3:
                w *= np.float32(scale / 128.0)  # the preprocessed input spans about +-128
            b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
            mods += [dict(type="conv", cin=cin, cout=cout, k=3, stride=1, pad=1, weight=w, bias=b), dict(type="relu")]
            cin = cout
        mods.append(dict(type="pool", kW=2, kH=2, dW=2, dH=2, padW=0, padH=0, ceil_mode=ceil_mode))
    return mods


def _module_codes(mods: Sequence[dict]) -> List[int]:
    codes = []
    for m in mods:
        if m["type"] == "conv":
            codes += [0, m["cin"], m["cout"], m["k"], m["stride"], m["pad"], 0, 0]
        elif m["type"] == "relu":
            codes += [1, 0, 0, 0, 0, 0, 0, 0]
        else:
            codes += [2, m["kW"], m["kH"], m["dW"], m["dH"], m["padW"], m["padH"], 1 if m["ceil_mode"] else 0]
    return codes


class PerceptualCriterion:
    """The loss network on the GPU.  `modules`: the dicts of t7.loss_network_from_model (at least up to the deepest layer)."""

    def __init__(self, modules: Sequence[dict], content_layers: Sequence, content_weights: Sequence[float],
                 style_layers: Sequence, style_weights: Sequence[float], agg_type: str = "gram"):
        if agg_type not in AGG_TYPES:
            raise ValueError(f"Unsupported aggregation type {agg_type}")  # StyleLoss.lua:23
        self.content_layers = [layer_index(s) for s in content_layers]
        self.style_layers = [layer_index(s) for s in style_layers]
        self.content_weights = [float(w) for w in content_weights]
        self.style_weights = [float(w) for w in style_weights]
        self.agg_type = agg_type
        if len(self.content_weights) != len(self.content_layers) or len(self.style_weights) != len(self.style_layers):
            raise ValueError("one weight per loss layer is needed (parse_layers repeats a single weight)")
        last = max(self.content_layers + self.style_layers)
        if last > len(modules):
            raise _lib.FavError(_lib.FAV_ERR_INVALID, f"loss network: layer {last} requested, the network has {len(modules)} modules")
        self.modules = list(modules[:last])  # trim_network (layer_utils.lua:146-165)
        codes = _module_codes(self.modules)
        ivec = lambda v: (C.c_int * max(1, len(v)))(*v)
        dvec = lambda v: (C.c_double * max(1, len(v)))(*v)
        h = C.c_void_p()
        _lib.check(_lib.lib.fav_percep_create(len(self.modules), ivec(codes), len(self.content_layers), ivec(self.content_layers),
                                              dvec(self.content_weights), len(self.style_layers), ivec(self.style_layers),
                                              dvec(self.style_weights), AGG_TYPES[agg_type], C.byref(h)))
        self._h = h
        try:
            for i, m in enumerate(self.modules, 1):
                if m["type"] == "conv":
                    w = np.ascontiguousarray(m["weight"], np.float32)
                    b = np.ascontiguousarray(m["bias"], np.float32)
                    _lib.check(_lib.lib.fav_percep_set_conv(h, i, w.ctypes.data_as(C.c_void_p), w.size, b.ctypes.data_as(C.c_void_p), b.size))
            _lib.check(_lib.lib.fav_percep_finalize(h))
        except Exception:
            self.close()
            raise

    @classmethod
    def from_t7(cls, path: str, content_layers, content_weights, style_layers, style_weights, agg_type: str = "gram"):
        from . import t7

        last = max(layer_index(s) for s in list(content_layers) + list(style_layers))
        return cls(t7.load_loss_network(path, last), content_layers, content_weights, style_layers, style_weights, agg_type)

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib.fav_percep_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    @staticmethod
    def _img(img: torch.Tensor) -> torch.Tensor:
        t = img.detach().reshape(3, img.shape[-2], img.shape[-1])
        return t.to(device="cuda", dtype=torch.float32).contiguous()

    def set_style_target(self, img: torch.Tensor) -> None:
        """setStyleTarget(preprocess(style_image)) (core.lua:93-97): img [3,H,W] RGB in [0,1], already scaled."""
        t = self._img(img)
        _lib.check(_lib.lib.fav_percep_set_style_target(self._h, _lib.dptr(t), t.shape[1], t.shape[2], _lib.stream_ptr()))

    def evaluate(self, content_img: torch.Tensor, stylized_img: torch.Tensor) -> Tuple[float, float]:
        """evaluate_image (core.lua:101-106) -> (total_content_loss, total_style_loss)."""
        a, b = self._img(content_img), self._img(stylized_img)
        if a.shape != b.shape:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, f"evaluate: content {tuple(a.shape)} and stylized {tuple(b.shape)} differ")
        cl, sl = C.c_double(), C.c_double()
        _lib.check(_lib.lib.fav_percep_evaluate(self._h, _lib.dptr(a), _lib.dptr(b), a.shape[1], a.shape[2], C.byref(cl), C.byref(sl),
                                                _lib.stream_ptr()))
        return cl.value, sl.value

    def layer_output(self, pass_: int, index: int) -> torch.Tensor:
        """Feature map of loss layer `index` from the last forward: pass 0 = content target, 1 = evaluated / style image."""
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        _lib.check(_lib.lib.fav_percep_layer_output(self._h, pass_, index, None, C.byref(c), C.byref(h), C.byref(w), None))
        out = torch.empty((c.value, h.value, w.value), device="cuda", dtype=torch.float32)
        _lib.check(_lib.lib.fav_percep_layer_output(self._h, pass_, index, _lib.dptr(out), None, None, None, _lib.stream_ptr()))
        return out

    def conv_output(self, module_index: int) -> torch.Tensor:
        """fp32 output of convolution module `module_index` (bias included, before ReLU / pooling) from the last forward()
        or backward() call: the values its ReLU masks and pooling arg-maxes were taken from.  [C,H,W] of the last image."""
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        _lib.check(_lib.lib.fav_percep_conv_output(self._h, module_index, None, C.byref(c), C.byref(h), C.byref(w), None))
        out = torch.empty((c.value, h.value, w.value), device="cuda", dtype=torch.float32)
        _lib.check(_lib.lib.fav_percep_conv_output(self._h, module_index, _lib.dptr(out), None, None, None, _lib.stream_ptr()))
        return out

    def forward(self, input: torch.Tensor, target) -> float:
        """percep_crit:forward(input, {content_target=...}) (PerceptualCriterion.lua:117-155, train_video.lua:343-344).

        input and target['content_target']: [N,3,H,W] (or [3,H,W]) in NET space, BGR 255 x - mean, as the training script
        feeds them; the style target is the one set_style_target captured.  Sets total_content_loss, total_style_loss,
        content_losses and style_losses (strength * MSE per layer) and returns their sum.  The gradient is computed in the same
        pass and returned by backward().  A batch is one call per image, scaled by 1/N: MSE over N*C*H*W for the content layers
        and over the N*C*C expanded target for the style layers (StyleLoss.lua:39-50) is the mean of the per-image losses."""
        x = self._batch(input)
        ct = target.get("content_target") if isinstance(target, dict) else target
        if isinstance(target, dict) and target.get("style_target") is not None:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "forward: set the style target with set_style_target (an RGB image)")
        if ct is None and self.content_layers:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "forward: the content layers need target['content_target']")
        ct = self._batch(ct) if ct is not None else None
        if ct is not None and ct.shape != x.shape:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, f"forward: input {tuple(x.shape)} and content target {tuple(ct.shape)} differ")
        N, _, H, W = x.shape
        nc, ns = len(self.content_layers), len(self.style_layers)
        grad = torch.empty_like(x)
        per = np.zeros(nc + ns)
        tc = ts = 0.0
        for n in range(N):
            cl, sl, lay = C.c_double(), C.c_double(), (C.c_double * max(1, nc + ns))()
            _lib.check(_lib.lib.fav_percep_forward_backward(self._h, _lib.dptr(ct[n]) if ct is not None else None, _lib.dptr(x[n]), H, W,
                                                            _lib.dptr(grad[n]), C.byref(cl), C.byref(sl), lay, _lib.stream_ptr()))
            tc += cl.value
            ts += sl.value
            per += np.asarray(lay[:nc + ns])
        if N > 1:
            grad.mul_(1.0 / N)
        self.total_content_loss, self.total_style_loss = tc / N, ts / N
        self.content_losses = [float(v) / N for v in per[:nc]]
        self.style_losses = [float(v) / N for v in per[nc:]]
        self.output = self.total_style_loss + self.total_content_loss
        self.gradInput = grad
        self._fb_args = (input, target)
        return self.output

    updateOutput = forward

    def backward(self, input: torch.Tensor, target) -> torch.Tensor:
        """percep_crit:backward(input, target) (PerceptualCriterion.lua:158-161): d output / d input, [N,3,H,W] net space."""
        args = getattr(self, "_fb_args", None)
        if args is None or args[0] is not input or args[1] is not target:
            self.forward(input, target)
        return self.gradInput

    updateGradInput = backward

    @staticmethod
    def _batch(img: torch.Tensor) -> torch.Tensor:
        t = img.detach().to(device="cuda", dtype=torch.float32)
        if t.dim() == 3:
            t = t[None]
        if t.dim() != 4 or t.shape[1] != 3:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, f"expected [N,3,H,W] images, got {tuple(img.shape)}")
        return t.contiguous()

    def style_stat(self, which: int, k: int) -> torch.Tensor:
        """Gram matrix [C,C] (or the C means) of style layer k: which 0 = style target, 1 = last evaluated image."""
        n = C.c_int()
        _lib.check(_lib.lib.fav_percep_style_stat(self._h, which, k, None, C.byref(n), None))
        out = torch.empty(n.value, device="cuda", dtype=torch.float64)
        _lib.check(_lib.lib.fav_percep_style_stat(self._h, which, k, _lib.dptr(out), None, _lib.stream_ptr()))
        if self.agg_type == "gram":
            c = int(round(n.value ** 0.5))
            out = out.reshape(c, c)
        return out


PIXEL_LOSS_TYPES = {"L2": 0, "L1": 1, "SmoothL1": 2}


def _nchw3(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.device.type != "cuda" or t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 4 or t.shape[1] != 3:
        raise _lib.FavError(_lib.FAV_ERR_INVALID, f"{what}: expected a contiguous CUDA float32 [N,3,H,W] tensor, got "
                                                  f"{tuple(t.shape)} {t.dtype} on {t.device}")
    return t


def pixel_loss_grad(out2: torch.Tensor, prev_warped_masked: torch.Tensor, cert: torch.Tensor, loss_type: str, weight: float,
                    grad_accum: torch.Tensor) -> float:
    """pixel_crit:forward / backward(out2 .* cert, out1_warped_masked) scaled by -pixel_loss_weight (train_video.lua:117-126,
    354-366): returns weight * loss and adds weight * d loss / d (out2 .* cert) to grad_accum in place, NOT multiplied by the
    certainty (the script adds the criterion's gradInput as it is).  out2, prev_warped_masked, grad_accum [N,3,H,W];
    cert [N,1,H,W]."""
    if loss_type not in PIXEL_LOSS_TYPES:
        raise ValueError(f"pixel loss type {loss_type!r}: L2, L1 or SmoothL1")
    N, _, H, W = _nchw3(out2, "out2").shape
    _nchw3(grad_accum, "grad_accum")
    prev = _nchw3(prev_warped_masked, "prev_warped_masked")
    if prev.shape != out2.shape or grad_accum.shape != out2.shape or tuple(cert.shape) != (N, 1, H, W):
        raise _lib.FavError(_lib.FAV_ERR_INVALID, "pixel_loss_grad: shape mismatch")
    c = cert.detach().to(device="cuda", dtype=torch.float32).contiguous()
    loss = C.c_double()
    _lib.check(_lib.lib.fav_pixel_loss_grad(_lib.dptr(out2), _lib.dptr(prev), _lib.dptr(c), N, H, W, PIXEL_LOSS_TYPES[loss_type],
                                            float(weight), _lib.dptr(grad_accum), C.byref(loss), _lib.stream_ptr()))
    return loss.value


def tv_grad(x: torch.Tensor, strength: float, grad_accum: torch.Tensor) -> torch.Tensor:
    """nn.TotalVariation(strength):updateGradInput(x, grad_accum) (TotalVariation.lua:19-35), in place on grad_accum."""
    N, _, H, W = _nchw3(x, "x").shape
    if _nchw3(grad_accum, "grad_accum").shape != x.shape:
        raise _lib.FavError(_lib.FAV_ERR_INVALID, "tv_grad: shape mismatch")
    _lib.check(_lib.lib.fav_tv_grad(_lib.dptr(x), N, H, W, float(strength), _lib.dptr(grad_accum), _lib.stream_ptr()))
    return grad_accum


def scale_style_image(img: torch.Tensor, size: int) -> torch.Tensor:
    """image.scale(style_image, opt.style_image_size) (fast_artistic_video_core.lua:94), on the host.  image.scale lives in the
    torch `image` rock, which is not vendored, so its arithmetic is NOT pinned: this reads a single size as the length of the
    longer side, the shorter side scaled in proportion and rounded, with bilinear interpolation (align_corners=True).  An image
    already at that size is returned unchanged."""
    _, H, W = img.shape
    if max(H, W) == size:
        return img
    if H >= W:
        oh, ow = size, max(1, int(round(W * size / H)))
    else:
        oh, ow = max(1, int(round(H * size / W))), size
    x = img.detach().to("cpu", torch.float32)[None]
    return torch.nn.functional.interpolate(x, size=(oh, ow), mode="bilinear", align_corners=True)[0]
