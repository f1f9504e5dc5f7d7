"""fast_artistic_video/models_video.lua -- `models_video.build_model(opt)` (:55-140).

Returns a StyleNet whose `forward(input[Nx7xHxW]) -> [Nx3xHxW]` runs the sm_90a path
(fav_net_forward_batch, include/fav.h).  Parameters are addressed by the names listed in fav.h.

Batches: like the reference nn modules, forward takes N >= 1 images of one size, and run_image / run_next_image /
run_next_image_flows accept a leading batch dimension.  A batch runs through one plan in one launch per kernel; image b of
the result is bit-identical to that image run alone.

Style banks (an addition): add_style(other) gives a net further weight sets of its architecture, and `styles=[s_0, ...]` on
forward / run_image / run_next_image / run_next_image_flows runs image b of a batch with style s_b -- bit-identical to that
image run alone on the net style s_b came from.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib, synth


class StyleNet:
    def __init__(self, arch: str = synth.DEFAULT_ARCH, padding_type: str = "reflect-start",
                 tanh_constant: float = 150.0, in_dim: int = 7, norm: str = "instance", precision: str = "pair"):
        """norm: 'instance' (InstanceNormalization, the default) or 'batch' (SpatialBatchNormalization in evaluate mode,
        -use_instance_norm 0; its parameters add '<n>.running_mean', '<n>.running_var' and '<n>.eps').
        precision: 'pair' (fp32 parity, the default) or 'fp16' (single pass; set_precision)."""
        h = C.c_void_p()
        _lib.check(_lib.lib.fav_net_create_norm(arch.encode(), padding_type.encode(), C.c_float(tanh_constant), in_dim,
                                                norm.encode(), C.byref(h)))
        self._h = h
        self.arch = arch
        self.in_dim = in_dim
        self.norm = norm
        self.finalized = False
        self.precision = "pair"
        if precision != "pair":
            self.set_precision(precision)

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

    def set_precision(self, mode: str) -> None:
        """'pair' (default): fp16 hi + lo operands, three MMAs per K step, fp32 parity.  'fp16': one MMA per K step on the hi
        halves, faster, about one 8-bit level off the exact frame (fav_net_set_precision).  An addition, not a reference
        option.  Drops the cached plans and graphs; frames in flight on a Session must be finished (Session.sync) first.
        The CUDA-core comparator (set_conv_impl('simt')) stays exact fp32."""
        _lib.check(_lib.lib.fav_net_set_precision(self._h, mode.encode()))
        self.precision = mode

    def add_style(self, other: "StyleNet") -> int:
        """Copy other's weights (its style 0) into this net as a new style and return its index (fav_net_add_style).  Both nets
        must be loaded and agree on arch, padding_type, tanh_constant, in_dim and norm (FavError naming the first that differs);
        at most 64 styles.  `other` may be dropped afterwards.  The bank runs in this net's precision.  Drops the cached plans
        and graphs."""
        idx = C.c_int()
        _lib.check(_lib.lib.fav_net_add_style(self._h, other._h, C.byref(idx)))
        return idx.value

    @property
    def num_styles(self) -> int:
        """Weight sets this net holds: 1 (its own) plus one per add_style."""
        return _lib.lib.fav_net_num_styles(self._h)

    def _set_styles(self, styles) -> None:
        """The style of each image of the next call (fav_net_set_batch_styles); None: style 0 for every image.  A sequence must
        have one entry per image of that call."""
        if styles is None:
            _lib.check(_lib.lib.fav_net_set_batch_styles(self._h, None, 0))
            return
        vals = [int(v) for v in styles]
        if not vals:
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "styles: an empty sequence (pass None for style 0 everywhere)")
        _lib.check(_lib.lib.fav_net_set_batch_styles(self._h, (C.c_int * len(vals))(*vals), len(vals)))

    def set_activation_budget(self, nbytes: int) -> None:
        """Cap the activation memory of plans (one per batch and frame size) created from now on; default 32 GiB.  A plan
        over the budget shares buffers between layers whose lifetimes do not overlap (same output, bit for bit); one over
        it even then is refused (FavError)."""
        _lib.check(_lib.lib.fav_net_set_activation_budget(self._h, int(nbytes)))

    def plan_bytes(self, H: int, W: int, batch: int = 1):
        """(all-live bytes, shared-arena bytes) of the activation buffers a plan for `batch` frames of H x W takes."""
        a, s = C.c_size_t(), C.c_size_t()
        _lib.check(_lib.lib.fav_net_plan_bytes(self._h, int(batch), int(H), int(W), C.byref(a), C.byref(s)))
        return a.value, s.value

    # -- model:forward(input) ----------------------------------------------------------------------
    def forward(self, input: torch.Tensor, styles=None) -> torch.Tensor:
        """styles: None (style 0), or the style of each of the N images (add_style)."""
        assert input.dim() == 4 and input.size(0) >= 1 and input.size(1) == self.in_dim, \
            f"expected Nx{self.in_dim}xHxW input"
        x = input.contiguous()
        assert x.dtype == torch.float32
        N, (H, W) = x.size(0), x.shape[-2:]
        out = torch.empty((N, 3, H, W), dtype=torch.float32, device=x.device)
        self._set_styles(styles)
        _lib.check(_lib.lib.fav_net_forward_batch(self._h, _lib.dptr(x), N, H, W, _lib.dptr(out), _lib.stream_ptr()))
        return out

    def profile(self, input: torch.Tensor):
        """One forward with per-step CUDA-event timing -> list of dict(kind, name, ms, work)."""
        x = input.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty((1, 3, H, W), dtype=torch.float32, device=x.device)
        self._set_styles(None)
        n_max = 256
        kinds, ms, work = (C.c_int * n_max)(), (C.c_float * n_max)(), (C.c_double * n_max)()
        names = C.create_string_buffer(24 * n_max)
        n = C.c_int()
        _lib.check(_lib.lib.fav_net_profile(self._h, _lib.dptr(x), H, W, _lib.dptr(out), n_max, kinds, ms, work, names,
                                            C.byref(n), _lib.stream_ptr()))
        kn = {0: "pack", 1: "conv", 2: "in_stats", 3: "in_apply"}
        return [dict(kind=kn[kinds[i]], name=names.raw[24 * i:24 * i + 24].split(b"\0")[0].decode(), ms=float(ms[i]),
                     work=float(work[i])) for i in range(n.value)]

    def layer_output(self, index: int, image: int = 0) -> torch.Tensor:
        """Activation after layer `index` of image `image` of the last forward's batch."""
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        _lib.check(_lib.lib.fav_net_layer_output_image(self._h, index, image, None, C.byref(c), C.byref(h), C.byref(w), None))
        out = torch.empty((c.value, h.value, w.value), dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib.fav_net_layer_output_image(self._h, index, image, _lib.dptr(out), C.byref(c), C.byref(h),
                                                       C.byref(w), _lib.stream_ptr()))
        return out

    # -- fused frame-level ops (fast_artistic_video_core.lua:121-180) ------------------------------------
    def run_image(self, img: torch.Tensor, fill: torch.Tensor = None, scale_factor: float = 1.0, styles=None) -> torch.Tensor:
        """img [3,H,W], or [B,3,H,W] for a batch (fill then [B,3,H,W] too).  styles: None (style 0), or one style per image
        (add_style; one entry for [3,H,W]).  scale_factor != 1 (-scale_factor, core.lua:127-152):
        one image [3,H,W] through an image model (in_dim 3), stylized at (H*sf) x (W*sf) between two bicubic image.scale
        calls (fav_run_image_scaled); fill is then unused, as it is for every image model."""
        x = img.contiguous()
        assert x.dim() in (3, 4) and x.size(-3) == 3 and x.dtype == torch.float32
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        self._set_styles(styles)
        if float(scale_factor) != 1:
            if x.dim() != 3:
                raise _lib.FavError(_lib.FAV_ERR_INVALID, f"run_image with scale_factor {scale_factor}: one image [3,H,W], "
                                    f"got {list(x.shape)}")
            _lib.check(_lib.lib.fav_run_image_scaled(self._h, _lib.dptr(x), H, W, C.c_double(float(scale_factor)),
                                                     _lib.dptr(out), _lib.stream_ptr()))
        elif x.dim() == 3:
            _lib.check(_lib.lib.fav_run_image(self._h, _lib.dptr(x), _lib.dptr(fill), H, W, _lib.dptr(out),
                                              _lib.stream_ptr()))
        else:
            fill = _planes(fill, x, 3)
            _lib.check(_lib.lib.fav_run_image_batch(self._h, _lib.dptr(x), _lib.dptr(fill), x.size(0), H, W, _lib.dptr(out),
                                                    _lib.stream_ptr()))
        return out

    def run_next_image(self, img, prev_rgb, flow, cert, fill=None, flow_mask=None,
                       border_mode=_lib.BORDER_PER_TAP, styles=None) -> torch.Tensor:
        """img / prev_rgb [3,H,W], flow [2,H,W], cert [H,W]; or all of them (and fill, flow_mask) with a leading batch
        dimension B: B independent clips advance one frame, each from its own prev_rgb[b].  styles: None (style 0), or one
        style per image (add_style)."""
        x = img.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        self._set_styles(styles)
        if x.dim() == 3:
            p, f, c = prev_rgb.contiguous(), flow.contiguous(), cert.contiguous()
            _lib.check(_lib.lib.fav_run_next_image(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(c),
                                                   _lib.dptr(fill), _lib.dptr(flow_mask), H, W, border_mode,
                                                   _lib.dptr(out), _lib.stream_ptr()))
        else:
            p, f, c = _planes(prev_rgb, x, 3), _planes(flow, x, 2), _planes(cert, x, 0)
            fill, flow_mask = _planes(fill, x, 3), _planes(flow_mask, x, 0)
            _lib.check(_lib.lib.fav_run_next_image_batch(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(c),
                                                         _lib.dptr(fill), _lib.dptr(flow_mask), x.size(0), H, W, border_mode,
                                                         _lib.dptr(out), _lib.stream_ptr()))
        return out


    def run_next_image_flows(self, img, prev_rgb, flow_bw, flow_fw_uv=None, cert_raw=None, min_filter_r=7, fill=None,
                             flow_mask=None, border_mode=_lib.BORDER_PER_TAP, styles=None) -> torch.Tensor:
        """run_next_image with func_load_cert + utils.min_filter inside (fav_run_next_image_flows): the whole temporal stage is
        ONE kernel.  flow_bw [2,H,W] (dy,dx); flow_fw_uv [2,H,W] (u,v) -> occlusion test on the GPU, or cert_raw [H,W].
        A leading batch dimension B on every argument: B independent clips advance one frame.  styles: None (style 0), or one
        style per image (add_style)."""
        x = img.contiguous()
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        self._set_styles(styles)
        if x.dim() == 3:
            p, f = prev_rgb.contiguous(), flow_bw.contiguous()
            fw = None if flow_fw_uv is None else flow_fw_uv.contiguous()
            cr = None if cert_raw is None else cert_raw.contiguous()
            _lib.check(_lib.lib.fav_run_next_image_flows(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(fw),
                                                         _lib.dptr(cr), _lib.dptr(fill), _lib.dptr(flow_mask), H, W,
                                                         int(min_filter_r), border_mode, _lib.dptr(out), _lib.stream_ptr()))
        else:
            p, f = _planes(prev_rgb, x, 3), _planes(flow_bw, x, 2)
            fw, cr = _planes(flow_fw_uv, x, 2), _planes(cert_raw, x, 0)
            fill, flow_mask = _planes(fill, x, 3), _planes(flow_mask, x, 0)
            _lib.check(_lib.lib.fav_run_next_image_flows_batch(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(fw),
                                                               _lib.dptr(cr), _lib.dptr(fill), _lib.dptr(flow_mask), x.size(0), H,
                                                               W, int(min_filter_r), border_mode, _lib.dptr(out),
                                                               _lib.stream_ptr()))
        return out

    def run_next_image_flows_structure(self, img, prev_rgb, flow_bw, flow_fw_uv, min_filter_r=7, fill=None, flow_mask=None,
                                       border_mode=_lib.BORDER_PER_TAP) -> torch.Tensor:
        """run_next_image_flows with the certainty in the checker's 4-argument mode, as the stylization scripts compute it
        (makeOptFlow_deepflow.sh:58-60): the structure term comes from img [3,H,W] (byte/255 values), the frame being stylized.
        flow_bw [2,H,W] (dy,dx), flow_fw_uv [2,H,W] (u,v).  One image."""
        x = img.contiguous()
        assert x.dim() == 3, "run_next_image_flows_structure: one image [3,H,W]"
        H, W = x.shape[-2:]
        out = torch.empty_like(x)
        self._set_styles(None)
        p, f, fw = prev_rgb.contiguous(), flow_bw.contiguous(), flow_fw_uv.contiguous()
        _lib.check(_lib.lib.fav_run_next_image_flows_structure(self._h, _lib.dptr(x), _lib.dptr(p), _lib.dptr(f), _lib.dptr(fw),
                                                               _lib.dptr(fill), _lib.dptr(flow_mask), H, W, int(min_filter_r),
                                                               border_mode, _lib.dptr(out), _lib.stream_ptr()))
        return out


def _planes(t, img, c):
    """t (or None) as a contiguous tensor of `c` planes per image of the batch img [B,3,H,W]; c = 0: one plane without a
    channel dimension ([B,H,W]; [B,1,H,W] is accepted as well).  Mismatched shapes raise
    FavError(FAV_ERR_INVALID) before anything is launched."""
    if t is None:
        return None
    lead, (H, W) = tuple(img.shape[:-3]), tuple(img.shape[-2:])
    want = lead + ((c,) if c else ()) + (H, W)
    if c == 0 and t.dim() == len(want) + 1 and t.size(-3) == 1:
        t = t.reshape(want)
    if tuple(t.shape) != want or t.dtype != torch.float32:
        raise _lib.FavError(_lib.FAV_ERR_INVALID, f"expected a float32 tensor of shape {list(want)}, got {t.dtype} {list(t.shape)}")
    return t.contiguous()


def build_model(opt) -> StyleNet:
    """M.build_model(opt) (models_video.lua:55): opt.arch, opt.padding_type, opt.tanh_constant, opt.use_instance_norm; and
    opt.precision ('pair' or 'fp16', StyleNet.set_precision), an addition."""
    get = (lambda k, d: opt.get(k, d)) if isinstance(opt, dict) else (lambda k, d: getattr(opt, k, d))
    return StyleNet(get("arch", synth.DEFAULT_ARCH), get("padding_type", "reflect-start"),
                    float(get("tanh_constant", 150.0)), norm="instance" if int(get("use_instance_norm", 1)) == 1 else "batch",
                    precision=get("precision", "pair"))


def synthetic_model(style: str = "candy", arch: str = synth.DEFAULT_ARCH, in_dim: int = 7, norm: str = "instance") -> StyleNet:
    """Seeded random-init weights for a named style (no network => no released checkpoints; SURVEY.md §8c).
    in_dim = 3: an image model (-model_img) of the same architecture."""
    return StyleNet(arch, in_dim=in_dim, norm=norm).load_state(synth.make_weights(arch, style, in_dim, norm))
