"""fast_artistic_video/models_video.lua -- `models_video.build_model(opt)` (:55-140).

Returns a StyleNet whose `forward(input[1x7xHxW]) -> [1x3xHxW]` runs the sm_90a path
(fav_net_forward, include/fav.h).  Parameters are addressed by the names listed in fav.h.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib, synth


class StyleNet:
    def __init__(self, arch: str = synth.DEFAULT_ARCH, padding_type: str = "reflect-start",
                 tanh_constant: float = 150.0, in_dim: int = 7):
        h = C.c_void_p()
        _lib.check(_lib.lib.fav_net_create(arch.encode(), padding_type.encode(), C.c_float(tanh_constant), in_dim,
                                           C.byref(h)))
        self._h = h
        self.arch = arch
        self.in_dim = in_dim
        self.finalized = False

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None and getattr(_lib, "lib", None) is not None:
            _lib.lib.fav_net_destroy(h)
            self._h = None

    # -- parameters ------------------------------------------------------------------------------
    def param_shapes(self) -> Dict[str, tuple]:
        out = {}
        name = C.create_string_buffer(64)
        shape = (C.c_int64 * 4)()
        numel = C.c_int64()
        for i in range(_lib.lib.fav_net_num_params(self._h)):
            _lib.check(_lib.lib.fav_net_param_info(self._h, i, name, shape, C.byref(numel)))
            shp = tuple(shape)
            n = name.value.decode()
            if n.endswith(".bias") or ".n" in n.rsplit(".", 1)[0][-3:]:
                shp = (shp[0],)
            out[n] = shp
        return out

    def load_state(self, weights: Dict[str, np.ndarray]) -> "StyleNet":
        for n in self.param_shapes():
            if n not in weights:
                raise KeyError(f"missing parameter {n}")
            a = np.ascontiguousarray(weights[n], dtype=np.float32)
            _lib.check(_lib.lib.fav_net_set_param(self._h, n.encode(), a.ctypes.data_as(C.c_void_p), a.size))
        _lib.check(_lib.lib.fav_net_finalize(self._h))
        self.finalized = True
        return self

    def set_conv_impl(self, impl: str) -> None:
        """'tcgen05' (default) or 'simt' (CUDA-core comparator used for bring-up / debugging)."""
        _lib.check(_lib.lib.fav_net_set_conv_impl(self._h, {"tcgen05": 0, "simt": 1}[impl]))

    # -- model:forward(input) ----------------------------------------------------------------------
    def forward(self, input: torch.Tensor) -> torch.Tensor:
        assert input.dim() == 4 and input.size(0) == 1 and input.size(1) == self.in_dim, \
            f"expected 1x{self.in_dim}xHxW input"
        x = input.contiguous()
        assert x.dtype == torch.float32
        H, W = x.shape[-2:]
        out = torch.empty((1, 3, H, W), dtype=torch.float32, device=x.device)
        _lib.check(_lib.lib.fav_net_forward(self._h, _lib.dptr(x), H, W, _lib.dptr(out), _lib.stream_ptr()))
        return out

    def profile(self, input: torch.Tensor):
        """One forward with per-step CUDA-event timing -> list of dict(kind, name, ms, work)."""
        x = input.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty((1, 3, H, W), dtype=torch.float32, device=x.device)
        n_max = 256
        kinds, ms, work = (C.c_int * n_max)(), (C.c_float * n_max)(), (C.c_double * n_max)()
        names = C.create_string_buffer(24 * n_max)
        n = C.c_int()
        _lib.check(_lib.lib.fav_net_profile(self._h, _lib.dptr(x), H, W, _lib.dptr(out), n_max, kinds, ms, work, names,
                                            C.byref(n), _lib.stream_ptr()))
        kn = {0: "pack", 1: "conv", 2: "in_stats", 3: "in_apply"}
        return [dict(kind=kn[kinds[i]], name=names.raw[24 * i:24 * i + 24].split(b"\0")[0].decode(), ms=float(ms[i]),
                     work=float(work[i])) for i in range(n.value)]

    def layer_output(self, index: int) -> torch.Tensor:
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        _lib.check(_lib.lib.fav_net_layer_output(self._h, index, None, C.byref(c), C.byref(h), C.byref(w), None))
        out = torch.empty((c.value, h.value, w.value), dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib.fav_net_layer_output(self._h, index, _lib.dptr(out), C.byref(c), C.byref(h), C.byref(w),
                                                 _lib.stream_ptr()))
        return out

    # -- fused frame-level ops (fast_artistic_video_core.lua:121-180) ------------------------------------
    def run_image(self, img: torch.Tensor, fill: torch.Tensor = None) -> torch.Tensor:
        x = img.contiguous()
        assert x.dim() == 3 and x.size(0) == 3 and x.dtype == torch.float32
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        _lib.check(_lib.lib.fav_run_image(self._h, _lib.dptr(x), _lib.dptr(fill), H, W, _lib.dptr(out),
                                          _lib.stream_ptr()))
        return out

    def run_next_image(self, img, prev_rgb, flow, cert, fill=None, flow_mask=None,
                       border_mode=_lib.BORDER_PER_TAP) -> torch.Tensor:
        x, p, f, c = img.contiguous(), prev_rgb.contiguous(), flow.contiguous(), cert.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        _lib.check(_lib.lib.fav_run_next_image(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(c),
                                               _lib.dptr(fill), _lib.dptr(flow_mask), H, W, border_mode,
                                               _lib.dptr(out), _lib.stream_ptr()))
        return out


    def run_next_image_flows(self, img, prev_rgb, flow_bw, flow_fw_uv=None, cert_raw=None, min_filter_r=7, fill=None,
                             flow_mask=None, border_mode=_lib.BORDER_PER_TAP) -> torch.Tensor:
        """run_next_image with func_load_cert + utils.min_filter inside (fav_run_next_image_flows): the whole temporal stage is
        ONE kernel.  flow_bw [2,H,W] (dy,dx); flow_fw_uv [2,H,W] (u,v) -> occlusion test on the GPU, or cert_raw [H,W]."""
        x, p, f = img.contiguous(), prev_rgb.contiguous(), flow_bw.contiguous()
        fw = None if flow_fw_uv is None else flow_fw_uv.contiguous()
        cr = None if cert_raw is None else cert_raw.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        _lib.check(_lib.lib.fav_run_next_image_flows(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(fw), _lib.dptr(cr),
                                                     _lib.dptr(fill), _lib.dptr(flow_mask), H, W, int(min_filter_r), border_mode,
                                                     _lib.dptr(out), _lib.stream_ptr()))
        return out


def build_model(opt) -> StyleNet:
    """M.build_model(opt) (models_video.lua:55): opt.arch, opt.padding_type, opt.tanh_constant, opt.use_instance_norm."""
    get = (lambda k, d: opt.get(k, d)) if isinstance(opt, dict) else (lambda k, d: getattr(opt, k, d))
    if int(get("use_instance_norm", 1)) != 1:
        raise _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, "use_instance_norm=0 (batch norm) is not on the inference path")
    return StyleNet(get("arch", synth.DEFAULT_ARCH), get("padding_type", "reflect-start"),
                    float(get("tanh_constant", 150.0)))


def synthetic_model(style: str = "candy", arch: str = synth.DEFAULT_ARCH, in_dim: int = 7) -> StyleNet:
    """Seeded random-init weights for a named style (no network => no released checkpoints; SURVEY.md §8c).
    in_dim = 3: an image model (-model_img) of the same architecture."""
    return StyleNet(arch, in_dim=in_dim).load_state(synth.make_weights(arch, style, in_dim))
