"""fast_artistic_video_vr.lua -- the 360-degree (cube-map) driver: six faces per frame in the order {6,1,2,5,3,4} (:103),
perspective border priors from already-stylized neighbour faces (:239-302), blend with the flow-warped previous frame,
re-blend of all six faces (:454-509), 3x3 median, cube map / equirectangular output (:511-559).

Every warp goes through nn.BilinearSamplerBDHW's replacement (fav_bilinear_sampler_bdhw_update_output); the per-face
re-blend is ONE fused kernel per face (fav_vr_blend_sides: 4 rotated gathers + combineSides + blend) instead of
4 warps + 4 rotations + 10 elementwise passes; the median runs on the GPU.  Mask algebra that happens once per stream
(init, :164-198) or on single-channel masks uses torch elementwise ops as plumbing.
-invert_occlusions / -fix_occlusions are parsed and ignored, exactly as in the reference (its VR func_load_cert, :204-237,
never reads them).

-evaluate (func_eval, :312-452) scores every face after it is saved: the gradient metric along the cut edges
(evaluate_gradient: six double sums from ONE kernel, fav_vr_eval_gradient), the seam MSE of the trimmed faces (evaluate_edge /
evaluate_edge_top, double-precision torch plumbing on O(S) elements), the content and style losses through the loss network
(core.make_evaluate_image; nan without one) and the temporal MSE (fav_temporal_mse).  The reference's quirks are kept: mode 3
compares the same face pair twice, evaluate_edge_top reads only its second argument (its 'top' term is 0), face 4's temporal
term sees prev_last_segments already replaced by this frame's re-blend, and -fix_occlusions_eval uses the VR script's own
per-pixel rule (:117-128).  The reference reads opt.reliable_map_min_filter without declaring it (:408-424); here it is an
option with train_video.lua's default 7.  Unequal overlaps are refused with -evaluate: the mode-4 MSE would compare slices of
different lengths (DESIGN.md section 8)."""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

from . import _lib, core, flowFileLoader, utils, vr_helper
from .video import flush_saves, load_image, save_image

PROC_ORDER = [6, 1, 2, 5, 3, 4]  # :103


def rotate90(t):  # reverse_tensor(t:transpose(2,3), 2)   :134-136
    return t.transpose(1, 2).flip(1).contiguous()


def rotateMinus90(t):  # :138-140
    return t.transpose(1, 2).flip(2).contiguous()


def rotate180(t):  # :142-144
    return t.flip(1).flip(2).contiguous()


_ROT = {None: 0, rotate90: 1, rotateMinus90: 2, rotate180: 3}


def getFormatedFlowFileName(pattern, fromIndex, toIndex, modeIdx):  # :108-115
    import re

    s = re.sub(r"\{(.*?)\}", lambda m: m.group(1) % fromIndex, pattern)
    s = re.sub(r"\[(.*?)\]", lambda m: m.group(1) % toIndex, s)
    return s % modeIdx


def gradient_ratios(sums, H, W):
    """gradx, grady, gradmag of evaluate_gradient (:375-386) from fav_vr_eval_gradient's six sums
    (sum gx, sum gy, sum MX, sum MY, sum gx*MX, sum gy*MY), with IEEE double semantics as Lua: 0/0 is nan, x/0 is inf."""
    Sgx, Sgy, Smx, Smy, Sgxm, Sgym = (np.float64(v) for v in sums)
    with np.errstate(divide="ignore", invalid="ignore"):
        gradx = (Sgxm / Smx) / (Sgx / np.float64(H * (W - 2)))
        grady = (Sgym / Smy) / (Sgy / np.float64((H - 2) * W))
        gradmag = (gradx * Smx + grady * Smy) / (Smx + Smy)
    return float(gradx), float(grady), float(gradmag)


def build_parser():
    p = argparse.ArgumentParser(prefix_chars="-")
    a = p.add_argument
    a("-input_pattern", default=""); a("-flow_pattern", default=""); a("-occlusions_pattern", default="")
    a("-model_img", default="self"); a("-model_vid", default="synthetic:mosaic")
    a("-start_frame", type=int, default=1); a("-continue_with", type=int, default=1); a("-num_frames", type=int, default=9999)
    a("-invert_occlusions", action="store_true"); a("-fix_occlusions", action="store_true")
    a("-occlusions_min_filter", type=int, default=7); a("-smooth_certainty", action="store_true")
    a("-fill_occlusions", default="vgg-mean"); a("-create_inconsistent", action="store_true")
    a("-create_inconsistent_border", action="store_true"); a("-backward", action="store_true")
    a("-overlap_pixel_w", type=int, default=20); a("-overlap_pixel_h", type=int, default=20)
    a("-output_prefix", default="out"); a("-out_equi_w", type=int, default=768); a("-out_equi_h", type=int, default=768)
    a("-out_equi", action="store_true"); a("-out_cubemap", action="store_true"); a("-median_filter", type=int, default=3)
    a("-gpu", type=int, default=0); a("-backend", default="cuda"); a("-use_cudnn", type=int, default=1)
    a("-cudnn_benchmark", type=int, default=0); a("-evaluate", action="store_true")
    # evaluation (:59-74); -loss_network names the .t7 loss network (without one, and no models/vgg16.t7, the perceptual rows are nan)
    a("-evaluation_file", default="evaluation.txt"); a("-no_consistency_eval", action="store_true")
    a("-flow_pattern_eval", default=""); a("-occlusions_pattern_eval", default="")
    a("-invert_occlusions_eval", action="store_true"); a("-backward_eval", action="store_true")
    a("-content_weights", default="1.0"); a("-content_layers", default="16"); a("-loss_network", default=None)
    a("-style_image", default=""); a("-style_image_size", type=int, default=256); a("-style_weights", default="5.0")
    a("-style_layers", default="4,9,16,23"); a("-style_target_type", default="gram", choices=["gram", "mean"])
    a("-fix_occlusions_eval", action="store_true")
    # read by func_eval (:408-424) but never declared by the VR script; train_video.lua:33's option and default
    a("-reliable_map_min_filter", type=int, default=7)
    a("-arch", default=core.synth.PAPER_ARCH)
    # not a reference option: "fp16" runs every convolution of the nets in one fp16 pass (fav_net_set_precision)
    a("-precision", default="pair", choices=["pair", "fp16"])
    return p


class VRDriver:
    def __init__(self, opt):
        self.opt = opt
        self.last_content = None
        self.last_segments = {}
        self.prev_last_segments = {}
        self.initialized = False
        self.outputs = {}  # file_idx -> dict(equi=..., cubemap=...) kept for callers / tests

    # ---- init (:164-198) ---------------------------------------------------------------------------------------
    def _init(self, hplus, wplus):
        opt, dev = self.opt, torch.device("cuda")
        assert hplus == wplus, "cube faces are square"
        self.hplus, self.wplus = hplus, wplus
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
        ones = torch.ones((1, hplus, wplus), device=dev)
        self.map = {"left": f32(vr_helper.make_perspective_warp_map_left(hplus, opt.overlap_pixel_w, wplus)),
                    "top": f32(vr_helper.make_perspective_warp_map_top(wplus, opt.overlap_pixel_h, hplus)),
                    "bottom": f32(vr_helper.make_perspective_warp_map_bottom(wplus, opt.overlap_pixel_h, hplus)),
                    "right": f32(vr_helper.make_perspective_warp_map_right(hplus, opt.overlap_pixel_w, wplus))}
        self.mask = {k: utils.warp_image(ones, v) for k, v in self.map.items()}
        msum = self.mask["left"] + self.mask["right"] + self.mask["top"] + self.mask["bottom"]
        self.mask_all_div = torch.clamp(msum, min=1)  # cmax(.,1)
        self.mask_all = torch.clamp(msum, max=1)      # cmin(.,1)
        gh, gw = opt.overlap_pixel_h - 10, opt.overlap_pixel_w - 10
        z = lambda h, w: np.zeros((h, w))
        col = lambda v: np.repeat(v[None, :], hplus, 0)   # values along w
        row = lambda v: np.repeat(v[:, None], wplus, 1)   # values along h
        g = {"left": np.concatenate([col(vr_helper.make_gradient_mask_w_dec(gw)), z(hplus, wplus - gw)], 1),
             "right": np.concatenate([z(hplus, wplus - gw), col(vr_helper.make_gradient_mask_w_inc(gw))], 1),
             "top": np.concatenate([row(vr_helper.make_gradient_mask_h_dec(gh)), z(hplus - gh, wplus)], 0),
             "bottom": np.concatenate([z(hplus - gh, wplus), row(vr_helper.make_gradient_mask_h_inc(gh))], 0)}
        g["all"] = np.maximum(np.maximum(g["left"], g["right"]), np.maximum(g["top"], g["bottom"]))
        g["left_right"] = np.maximum(g["left"], g["right"])
        self.grad = {k: f32(v)[None] for k, v in g.items()}
        self.anti_all = f32(1.0 - g["all"])  # csub(ones, grad_mask_all) in DOUBLE, then :type(dtype)  (:456)
        if opt.out_equi:
            r = opt.median_filter // 2
            self.equi_map = f32(vr_helper.make_cube_to_equirectangular_map(hplus - 2 * r, wplus - 2 * r, opt.overlap_pixel_w - r,
                                                                         opt.overlap_pixel_h - r, opt.out_equi_w, opt.out_equi_h))
        if opt.evaluate:  # the min-filtered masks of evaluate_gradient (:408-424), indexed by mode
            rr = opt.reliable_map_min_filter
            mf = lambda m: (utils.min_filter(m, rr) if rr > 1 else m)[0].contiguous()
            self.eval_mask = {1: mf(self.mask["left"]), 2: mf(self.mask["right"]), 3: mf(self.mask["right"] + self.mask["left"]),
                              4: mf(self.mask_all)}
            self.eval_mask[5] = self.eval_mask[4]
        self.initialized = True

    # ---- callbacks ---------------------------------------------------------------------------------------------
    def func_load_image(self, opt, i, dtype):  # :154-201
        mode, file_idx = (i - 1) % 6, (i - 1) // 6 + opt.start_frame
        path = opt.input_pattern % (file_idx, PROC_ORDER[mode])
        if not utils.file_exists(path):
            return None
        img = load_image(path, 3)
        if not self.initialized:
            self._init(img.shape[1], img.shape[2])
        self.last_content = img.contiguous()  # :200, the content image of func_eval's perceptual term
        return self.last_content

    def func_load_cert(self, opt, i, dtype):  # :204-237
        mode, file_idx = (i - 1) % 6, (i - 1) // 6 + opt.start_frame
        cert_border = torch.zeros((1, self.hplus, self.wplus), device="cuda")
        if not opt.create_inconsistent_border:
            if mode in (1, 3, 4, 5):
                cert_border = torch.maximum(cert_border, self.mask["left"])
            if mode in (2, 3, 4, 5):
                cert_border = torch.maximum(cert_border, self.mask["right"])
            if mode in (4, 5):
                cert_border = torch.maximum(torch.maximum(cert_border, self.mask["top"]), self.mask["bottom"])
        if i >= 7 and not opt.create_inconsistent:
            name = getFormatedFlowFileName(opt.occlusions_pattern, file_idx - 1, file_idx, PROC_ORDER[mode])
            utils.wait_for_file(name)
            return torch.maximum(load_image(name, 1).cuda(), cert_border)
        return cert_border

    def _warp(self, seg, which, rot=None):
        return utils.warp_image(rot(seg) if rot else seg, self.map[which])

    def func_make_last_frame_warped(self, opt, i, dtype, cert):  # :239-302
        mode, file_idx = (i - 1) % 6, (i - 1) // 6 + opt.start_frame
        ls, div = self.last_segments, self.mask_all_div
        border = torch.zeros((3, self.hplus, self.wplus), device="cuda")
        gradMask = None
        if not opt.create_inconsistent_border:
            if mode == 1:
                border, gradMask = self._warp(ls[1], "left"), self.grad["right"]
            elif mode == 2:
                border, gradMask = self._warp(ls[1], "right"), self.grad["left"]
            elif mode == 3:
                border = self._warp(ls[2], "left") + self._warp(ls[3], "right")
                gradMask = self.grad["left_right"]
            elif mode == 4:
                border = (self._warp(ls[2], "left", rotate90) / div + self._warp(ls[3], "right", rotateMinus90) / div +
                          self._warp(ls[4], "top") / div + self._warp(ls[1], "bottom", rotate180) / div)
                gradMask = self.grad["all"]
            elif mode == 5:
                border = (self._warp(ls[2], "left", rotateMinus90) / div + self._warp(ls[3], "right", rotate90) / div +
                          self._warp(ls[1], "top", rotate180) / div + self._warp(ls[4], "bottom") / div)
                gradMask = self.grad["all"]
        if i >= 7 and not opt.create_inconsistent:
            name = getFormatedFlowFileName(opt.flow_pattern, file_idx - 1, file_idx, PROC_ORDER[mode])
            utils.wait_for_file(name)
            flow = torch.from_numpy(flowFileLoader.load(name)).cuda()
            last_frame_warped = utils.warp_image(self.prev_last_segments[mode + 1], flow)
            if mode == 0:
                result = last_frame_warped
            else:
                cert_inv = 1.0 - cert.reshape(1, self.hplus, self.wplus)
                grad_mask = [self.grad["right"], self.grad["left"], self.grad["left_right"], self.grad["all"], self.grad["all"]][mode - 1]
                masks = [self.mask["left"], self.mask["right"], self.mask["left"] + self.mask["right"], self.mask_all, self.mask_all][mode - 1]
                mask = torch.maximum(grad_mask, torch.ceil(grad_mask) * cert_inv) * masks  # :288
                result = last_frame_warped * (1.0 - mask) + border * mask                  # :289-290
        else:
            result = border
        if opt.smooth_certainty and gradMask is None:
            # :297 indexes gradMask, which is nil for face 6 (mode 0) and with -create_inconsistent_border: the reference
            # raises a Lua error here, i.e. -smooth_certainty only works together with -create_inconsistent
            raise _lib.FavError(_lib.FAV_ERR_INVALID, "-smooth_certainty: no gradient mask for this face (gradMask is nil, "
                                "fast_artistic_video_vr.lua:245,297); use it with -create_inconsistent")
        if opt.smooth_certainty:  # :296-297
            return result, torch.clamp(torch.sign(torch.clamp(gradMask - 0.5, min=0.0)), min=0.25)
        return result

    def func_is_single_image(self, i, opt):  # :304-310
        return i % 6 == 1 if opt.create_inconsistent else i == 1

    # ---- -evaluate (:312-452) ----------------------------------------------------------------------------------------
    def _trim(self, t):  # :321-325
        oh, ow = self.opt.overlap_pixel_h // 2, self.opt.overlap_pixel_w // 2
        return t[:, oh:self.hplus - oh, ow:self.wplus - ow]

    @staticmethod
    def _mse(a, b):  # nn.MSECriterion (mean), in double on the device
        return float(((a.double() - b.double()) ** 2).mean())

    def _edge(self, img1, img2):  # evaluate_edge(img1, img2, 'left') (:312-319)
        return self._mse(img1[:, :, :1], img2[:, :, -1:])

    def _edge_top(self, img2, edgeOther):  # evaluate_edge_top (:327-341): its first argument is never read
        side1 = img2[:, :1, :]
        if edgeOther == "left":
            side2 = img2[:, :, :1].transpose(1, 2)
        elif edgeOther == "right":
            side2 = img2[:, :, -1:].transpose(1, 2).flip(2)
        elif edgeOther == "top":
            side2 = img2[:, :1, :].flip(1)  # reverses a size-1 dimension: side2 == side1
        else:
            side2 = img2[:, -1:, :]
        return self._mse(side1, side2)

    def _gradient(self, face, mask):  # evaluate_gradient (:344-387)
        H, W = face.shape[-2:]
        sums = torch.empty(6, dtype=torch.float64, device=face.device)
        _lib.check(_lib.lib.fav_vr_eval_gradient(_lib.dptr(face.contiguous()), _lib.dptr(mask), H, W, _lib.dptr(sums),
                                                 _lib.stream_ptr()))
        return gradient_ratios(sums.tolist(), H, W)

    def _load_flow_cert_eval(self, opt, file_idx, mode):  # load_flow_cert_eval (:389-401)
        name = lambda pat: getFormatedFlowFileName(pat, file_idx - 1, file_idx, PROC_ORDER[mode])
        flow = torch.from_numpy(flowFileLoader.load(name(opt.flow_pattern_eval or opt.flow_pattern))).cuda()
        cert = load_image(name(opt.occlusions_pattern_eval or opt.occlusions_pattern), 1).cuda()
        if opt.invert_occlusions_eval:
            cert = 1.0 - cert
        if opt.fix_occlusions_eval:  # fix_occlusions (:117-128): the displacement itself is tested against [0,H] x [0,W]
            H, W = flow.shape[-2:]
            out = (flow[0] < 0) | (flow[0] > H) | (flow[1] < 0) | (flow[1] > W)
            cert = cert.masked_fill(out[None], 0.0)
        return flow, cert

    def func_eval(self, opt, i, func_percept_loss, dtype):  # :403-452
        mode, file_idx = (i - 1) % 6, (i - 1) // 6 + 1  # file_idx without opt.start_frame, as written (:405)
        ls = self.last_segments
        gradx = grady = gradmag = edge = 0.0
        if mode != 0:
            gradx, grady, gradmag = self._gradient(ls[mode + 1], self.eval_mask[mode])
        if mode == 1:
            edge = self._edge(self._trim(ls[1]), self._trim(ls[2]))
        elif mode == 2:
            edge = self._edge(self._trim(ls[3]), self._trim(ls[1]))
        elif mode == 3:  # the same pair twice (:415-416)
            edge = (self._edge(self._trim(ls[2]), self._trim(ls[4])) + self._edge(self._trim(ls[2]), self._trim(ls[4]))) / 2
        elif mode == 4:  # every term reads trim(last_segments[5]) only (:419-422)
            t5 = self._trim(ls[5])
            edge = (self._edge_top(t5, "top") + self._edge_top(t5, "right") + self._edge_top(t5, "left")
                    + self._edge_top(t5, "bottom")) / 4
        # (content, style) unpacked as `style_loss, content_loss` (:427), as in the plain driver; nan without a loss network
        nan = float("nan")
        style_loss, content_loss = func_percept_loss(self.last_content, ls[mode + 1]) if func_percept_loss else (nan, nan)
        if i > 6 and not opt.no_consistency_eval:
            flow, cert = self._load_flow_cert_eval(opt, file_idx, mode)
            # at mode 5 func_save_image has already replaced prev_last_segments with this frame's re-blend (:530-532)
            if opt.backward_eval:
                t = utils.temporal_loss(ls[mode + 1], self.prev_last_segments[mode + 1], flow, cert)
            else:
                t = utils.temporal_loss(self.prev_last_segments[mode + 1], ls[mode + 1], flow, cert)
            return [gradx, grady, gradmag, edge, style_loss, content_loss, t], 7
        if opt.no_consistency_eval:
            return [gradx, grady, gradmag, edge, style_loss, content_loss], 6
        return [gradx, grady, gradmag, edge, style_loss, content_loss, 0.0], 7

    def blend_other_sides(self):  # :454-509 -- one fused kernel per face
        ls = self.last_segments
        plan = {1: [(2, "right", None), (3, "left", None), (5, "bottom", rotate180), (6, "top", rotate180)],
                2: [(1, "left", None), (4, "right", None), (5, "bottom", rotateMinus90), (6, "top", rotate90)],
                3: [(1, "right", None), (4, "left", None), (5, "bottom", rotate90), (6, "top", rotateMinus90)],
                4: [(2, "left", None), (3, "right", None), (5, "bottom", None), (6, "top", None)],
                5: [(1, "bottom", rotate180), (2, "left", rotate90), (3, "right", rotateMinus90), (4, "top", None)],
                6: [(1, "top", rotate180), (2, "left", rotateMinus90), (3, "right", rotate90), (4, "bottom", None)]}
        out = {}
        S = self.hplus
        for face, sides in plan.items():
            o = torch.empty_like(ls[face])
            imgs = (C.c_void_p * 4)(*[ls[s].data_ptr() for s, _, _ in sides])
            maps = (C.c_void_p * 4)(*[self.map[m].data_ptr() for _, m, _ in sides])
            rots = (C.c_int * 4)(*[_ROT[r] for _, _, r in sides])
            _lib.check(_lib.lib.fav_vr_blend_sides(_lib.dptr(ls[face]), imgs, maps, rots, _lib.dptr(self.mask_all_div),
                                                   _lib.dptr(self.grad["all"]), _lib.dptr(self.anti_all), _lib.dptr(o), S,
                                                   _lib.stream_ptr()))
            out[face] = o
        return out

    def func_save_image(self, opt, i, frame, dtype=None):  # :511-559
        mode, file_idx = (i - 1) % 6, (i - 1) // 6 + 1
        self.last_segments[mode + 1] = frame.contiguous()
        if mode != 5:
            return
        self.prev_last_segments = self.blend_other_sides()
        sides = {j: (utils.median_filter(self.prev_last_segments[j], opt.median_filter) if opt.median_filter > 0
                     else self.prev_last_segments[j]) for j in range(1, 7)}
        ow = opt.overlap_pixel_w // 2 - opt.median_filter // 2
        oh = opt.overlap_pixel_h // 2 - opt.median_filter // 2
        res = {}
        d = os.path.dirname(opt.output_prefix)
        if d and not os.path.isdir(d):
            os.makedirs(d)
        if opt.out_equi:
            strip = torch.cat([sides[1], sides[2], sides[3], sides[4], rotate180(sides[5]), rotate180(sides[6])], 2)
            res["equi"] = utils.warp_image(strip.contiguous(), self.equi_map)
            save_image("%s-%05d_equi.png" % (opt.output_prefix, file_idx), res["equi"], background=True)
        if opt.out_cubemap:
            # :548-553: {oversize+1, hplus-oversize} index the MEDIAN-FILTERED face (already 2*(r//2) smaller), so each
            # face comes out (hplus - overlap + 2*(r//2)) wide -- the reference's own (asymmetric) crop, kept as is
            crop = lambda t: t[:, oh:self.hplus - oh, ow:self.wplus - ow]
            res["cubemap"] = torch.cat([crop(sides[4]), crop(sides[1]), rotate90(crop(sides[5])), rotateMinus90(crop(sides[6])),
                                        crop(sides[3]), crop(sides[2])], 2)
            save_image("%s-%05d_cubemap.png" % (opt.output_prefix, file_idx), res["cubemap"], background=True)
        self.outputs[file_idx] = res


def main(argv=None, model_vid=None):
    opt = build_parser().parse_args(argv)
    if opt.input_pattern == "":
        raise SystemExit("Must give -input_pattern")
    if not opt.create_inconsistent and (opt.flow_pattern == "" or opt.occlusions_pattern == ""):
        raise SystemExit("Must give -flow_pattern and -occlusions_pattern")
    opt.num_frames = opt.num_frames * 6  # :574
    opt.scale_factor = 1
    if opt.continue_with > 1:
        # :576-584 reloads prev_last_segments from "<prefix><n>_<mode>.png", files whose image.save is commented out in
        # the reference itself (:524-526): the branch cannot work there either.
        raise _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, "-continue_with > 1: the reference reloads per-face PNGs it never "
                            "writes (fast_artistic_video_vr.lua:524-526,576-584)")
    if opt.overlap_pixel_w % 2 or opt.overlap_pixel_h % 2:
        raise _lib.FavError(_lib.FAV_ERR_INVALID, "overlap_pixel_w/h must be even (the reference slices with overlap/2, :515-516)")
    if opt.evaluate and opt.overlap_pixel_w != opt.overlap_pixel_h:
        # evaluate_edge_top's MSECriterion compares a trimmed row with a trimmed column (:419-422): equal lengths only
        raise _lib.FavError(_lib.FAV_ERR_INVALID, "-evaluate needs overlap_pixel_w == overlap_pixel_h (the mode-4 seam MSE compares "
                            "a trimmed row with a trimmed column, fast_artistic_video_vr.lua:327-341,419-422)")
    d = VRDriver(opt)
    core.run_fast_neural_video(opt, d.func_load_image, d.func_load_cert, d.func_eval, d.func_make_last_frame_warped,
                               d.func_is_single_image, d.func_save_image, model_vid=model_vid)
    torch.cuda.synchronize()
    flush_saves()  # the PNGs of a VR frame are encoded on worker threads while the next frame's faces are stylized
    return d


if __name__ == "__main__":
    main(sys.argv[1:])
