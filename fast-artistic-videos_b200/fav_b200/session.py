"""Host-buffer frame loop (fav_session_*, include/fav.h): the reference-facing call whose e2e time bench.py reports."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .models_video import StyleNet


def _hp(a):
    if isinstance(a, torch.Tensor):
        assert not a.is_cuda and a.is_contiguous() and a.dtype == torch.float32
        return C.c_void_p(a.data_ptr())
    assert isinstance(a, np.ndarray) and a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class Session:
    def __init__(self, net: StyleNet, H: int, W: int):
        h = C.c_void_p()
        _lib.check(_lib.lib.fav_session_create(net._h, H, W, C.byref(h)))
        self._h, self.net, self.H, self.W = h, net, H, W

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None and getattr(_lib, "lib", None) is not None:
            _lib.lib.fav_session_destroy(h)
            self._h = None

    def set_image_model(self, net_img: StyleNet = None):
        """-model_img: single images go through a separate 3-channel image model (None = 'self')."""
        _lib.check(_lib.lib.fav_session_set_image_model(self._h, net_img._h if net_img is not None else None))
        self.net_img = net_img  # keep it alive

    def run_image(self, content_host, out_host):
        _lib.check(_lib.lib.fav_session_run_image(self._h, _hp(content_host), _hp(out_host)))

    def run_next_image(self, content_host, flow_host, cert_host, out_host, min_filter_r=7,
                       border_mode=_lib.BORDER_PER_TAP):
        _lib.check(_lib.lib.fav_session_run_next_image(self._h, _hp(content_host), _hp(flow_host), _hp(cert_host),
                                                       int(min_filter_r), border_mode, _hp(out_host)))

    def run_next_image_flows(self, content_host, flow_bw_uv_host, flow_fw_uv_host, out_host, min_filter_r=7,
                             border_mode=_lib.BORDER_PER_TAP):
        _lib.check(_lib.lib.fav_session_run_next_image_flows(self._h, _hp(content_host), _hp(flow_bw_uv_host),
                                                             _hp(flow_fw_uv_host), int(min_filter_r), border_mode,
                                                             _hp(out_host)))

    def run_next_image_flows_structure(self, content_host, flow_bw_uv_host, flow_fw_uv_host, out_host, min_filter_r=7,
                                       border_mode=_lib.BORDER_PER_TAP):
        """run_next_image_flows with the certainty in the checker's 4-argument mode (structure term from the frame)."""
        _lib.check(_lib.lib.fav_session_run_next_image_flows_structure(self._h, _hp(content_host), _hp(flow_bw_uv_host),
                                                                       _hp(flow_fw_uv_host), int(min_filter_r), border_mode,
                                                                       _hp(out_host)))

    def run_frame_bytes(self, rgb_hwc, flo_uv, cert8, rows_out, invert_occlusion=False, min_filter_r=7,
                        border_mode=_lib.BORDER_PER_TAP):
        """One frame from file payloads (uint8 HWC frame, float32 [H,W,2] (u,v) flow, uint8 certainty; the last two None for
        the first frame); rows_out: uint8 [H, 1+3W] receives the Sub-filtered PNG scanlines of the stylized frame."""
        bp = lambda a: None if a is None else C.c_void_p(a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data)
        _lib.check(_lib.lib.fav_session_run_frame_bytes(self._h, bp(rgb_hwc), bp(flo_uv), bp(cert8), 1 if invert_occlusion else 0,
                                                        int(min_filter_r), border_mode, bp(rows_out)))

    def run_frame_bytes_flows(self, rgb_hwc, flo_bw_uv, flo_fw_uv, rows_out, min_filter_r=7, border_mode=_lib.BORDER_PER_TAP):
        """run_frame_bytes with the backward and forward .flo payloads (float32 [H,W,2] (u,v); both None for the first frame)
        instead of a certainty: the certainty is the checker's 4-argument mode with this frame, computed on the GPU."""
        bp = lambda a: None if a is None else C.c_void_p(a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data)
        _lib.check(_lib.lib.fav_session_run_frame_bytes_flows(self._h, bp(rgb_hwc), bp(flo_bw_uv), bp(flo_fw_uv), int(min_filter_r),
                                                              border_mode, bp(rows_out)))

    def frame_done(self, frame_index: int, wait: bool = True) -> bool:
        """The output of the frame_index-th run_* call (0-based) has landed in its host buffer."""
        rc = _lib.lib.fav_session_frame_done(self._h, int(frame_index), 1 if wait else 0)
        if rc == _lib.FAV_OK:
            return True
        if not wait and rc == _lib.FAV_ERR_INVALID:
            return False
        _lib.check(rc)
        return False

    def sync(self):
        _lib.check(_lib.lib.fav_session_sync(self._h))

    def last_gpu_ms(self) -> float:
        return float(_lib.lib.fav_session_last_gpu_ms(self._h))
