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
