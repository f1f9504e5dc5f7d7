"""fp64 numpy restatement of the VR driver's -evaluate (fast_artistic_video_vr.lua:117-128, 312-452), statement by statement,
quirks included, plus an evaluation hook for oracle/vr_oracle.py's driver restatement (VRRef / run_vr_clip).  TEST
INFRASTRUCTURE ONLY.  The gradient metric is in double from the fp32 face and the fp32 min-filtered mask, as the reference
computes it after :double(); the seam MSEs are taken in double here (the reference's CudaTensor criterion is fp32)."""
from __future__ import annotations

import numpy as np

from oracle import pyoracle, vr_oracle


def reverse_tensor(t, n):  # :130-132 (n is 1-based)
    return np.flip(t, axis=n - 1)


def mse(a, b):
    """nn.MSECriterion (sizeAverage): both inputs in logical order; element counts must agree (THNN's check)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.size != b.size:
        raise ValueError(f"MSECriterion: input and target have {a.size} and {b.size} elements")
    return float(np.mean((a.ravel() - b.ravel()) ** 2))


def trim(t, overlap_w, overlap_h):  # :321-325: {oversize+1, size-oversize} are 1-based inclusive
    H, W = t.shape[-2:]
    oh, ow = overlap_h // 2, overlap_w // 2
    return t[:, oh:H - oh, ow:W - ow]


def evaluate_edge(img1, img2, edge):  # :312-319
    if edge == "left":
        return mse(img1[:, :, 0:1], img2[:, :, img2.shape[2] - 1:])
    elif edge == "top":
        return mse(img1[:, 0:1, :], img2[:, img2.shape[1] - 1:, :])


def evaluate_edge_top(img1, img2, edgeOther):  # :327-341 -- img1 is never read
    side1 = img2[:, 0:1, :]
    side2 = None
    if edgeOther == "left":
        side2 = np.swapaxes(img2[:, :, 0:1], 1, 2)
    elif edgeOther == "right":
        side2 = reverse_tensor(np.swapaxes(img2[:, :, img2.shape[2] - 1:], 1, 2), 3)
    elif edgeOther == "top":
        side2 = reverse_tensor(img2[:, 0:1, :], 2)  # dimension 2 has size 1: a no-op
    elif edgeOther == "bottom":
        side2 = img2[:, img2.shape[1] - 1:, :]
    return mse(side1, side2)


def _conv_x(p):  # torch.conv2(p, {{-1,0,1}}, 'V'): a true convolution, the kernel is flipped
    return p[:, 0:-2] * 1.0 + p[:, 1:-1] * 0.0 + p[:, 2:] * -1.0


def _conv_y(p):  # torch.conv2(p, {{-1},{0},{1}}, 'V')
    return p[0:-2, :] * 1.0 + p[1:-1, :] * 0.0 + p[2:, :] * -1.0


def _maxpool3(p):  # nn.SpatialMaxPooling(3, 3, 1, 1, 1, 1): padding cells never win
    H, W = p.shape
    q = np.pad(p, 1, mode="constant", constant_values=-np.inf)
    return np.max(np.stack([q[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)]), axis=0)


def gradient_sums(img, mask):
    """The six sums evaluate_gradient (:344-387) divides: gradient_x:sum(), gradient_y:sum(), mask_gradient_x:sum(),
    mask_gradient_y:sum(), masked_gradient_x:sum(), masked_gradient_y:sum().  img [3,H,W] fp32, mask [1,H,W] (min-filtered)."""
    img = np.asarray(img, np.float32)
    d = [img[c].astype(np.float64) for c in range(3)]                                              # img[c]:double()
    gradient_x = np.maximum(np.maximum(np.abs(_conv_x(d[0])), np.abs(_conv_x(d[1]))), np.abs(_conv_x(d[2])))
    gradient_y = np.maximum(np.maximum(np.abs(_conv_y(d[0])), np.abs(_conv_y(d[1]))), np.abs(_conv_y(d[2])))
    m = np.asarray(mask, np.float32).astype(np.float64)[0]                                         # :double(), mask[1]
    mask_gradient_x = _maxpool3(np.abs(_conv_x(m)))
    mask_gradient_y = _maxpool3(np.abs(_conv_y(m)))
    masked_gradient_x = gradient_x * mask_gradient_x
    masked_gradient_y = gradient_y * mask_gradient_y
    return [float(gradient_x.sum()), float(gradient_y.sum()), float(mask_gradient_x.sum()), float(mask_gradient_y.sum()),
            float(masked_gradient_x.sum()), float(masked_gradient_y.sum())]


def gradient_ratios(sums, H, W):  # :375-386 in IEEE double: 0/0 is nan, x/0 is inf, as in Lua
    gx, gy, mx, my, gxm, gym = (np.float64(v) for v in sums)
    with np.errstate(divide="ignore", invalid="ignore"):
        gradx_per_pixel_full = gx / np.float64(H * (W - 2))
        grady_per_pixel_full = gy / np.float64((H - 2) * W)
        gradx_per_pixel_masked = gxm / mx
        grady_per_pixel_masked = gym / my
        gradx_ratio, grady_ratio = gradx_per_pixel_masked / gradx_per_pixel_full, grady_per_pixel_masked / grady_per_pixel_full
        gradmag_ratio = (gradx_ratio * mx + grady_ratio * my) / (mx + my)
    return float(gradx_ratio), float(grady_ratio), float(gradmag_ratio)


def evaluate_gradient(img, mask):
    H, W = img.shape[-2:]
    return gradient_ratios(gradient_sums(img, mask), H, W)


def fix_occlusions(flow, disoccluded):  # :117-128 (flow in the Lua loader's (dy, dx) layout), in place
    H, W = flow.shape[1], flow.shape[2]
    for x in range(W):
        for y in range(H):
            if flow[0][y][x] < 0 or flow[0][y][x] > H or flow[1][y][x] < 0 or flow[1][y][x] > W:
                disoccluded[0][y][x] = 0


class VREval:
    """func_eval (:403-452) over the state of a VRRef.  eval_flows[f][face] / eval_certs[f][face] are what
    load_flow_cert_eval reads for VR frame f (0-based) before -invert_occlusions_eval / -fix_occlusions_eval; percept is
    (content, stylized) -> (content_loss, style_loss) or None (the perceptual terms are then nan)."""

    def __init__(self, ref, frames, eval_flows, eval_certs, reliable_map_min_filter=7, no_consistency_eval=False,
                 backward_eval=False, invert_occlusions_eval=False, fix_occlusions_eval=False, percept=None):
        self.ref, self.frames, self.eval_flows, self.eval_certs = ref, frames, eval_flows, eval_certs
        self.no_consistency_eval, self.backward_eval = no_consistency_eval, backward_eval
        self.invert, self.fix, self.percept = invert_occlusions_eval, fix_occlusions_eval, percept
        r = reliable_map_min_filter
        mf = lambda m: (pyoracle.min_filter(m[0], r)[None] if r > 1 else m).astype(np.float64)  # utils.min_filter(...):double()
        self.mask_left, self.mask_right = mf(ref.mask_left), mf(ref.mask_right)
        self.mask_left_right = mf((ref.mask_right + ref.mask_left).astype(np.float32))              # torch.add(mask_right, mask_left)
        self.mask_all = mf(ref.mask_all)

    def _trim(self, t):
        return trim(t, self.ref.ow, self.ref.oh)

    def load_flow_cert_eval(self, f, mode):  # :389-401
        face = vr_oracle.PROC_ORDER[mode]
        flow_eval = np.array(self.eval_flows[f][face], np.float32)
        cert_eval = np.array(self.eval_certs[f][face], np.float32).reshape(1, *flow_eval.shape[1:])
        if self.invert:
            cert_eval = (np.float32(1) - cert_eval).astype(np.float32)
        if self.fix:
            fix_occlusions(flow_eval, cert_eval)
        return flow_eval, cert_eval

    def __call__(self, i):
        ref, ls = self.ref, self.ref.last_segments
        mode = (i - 1) % 6
        f = (i - 1) // 6
        tr = self._trim
        gradx, grady, gradmag, edge = 0.0, 0.0, 0.0, 0.0
        if mode == 1:
            gradx, grady, gradmag = evaluate_gradient(ls[2], self.mask_left)
            edge = evaluate_edge(tr(ls[1]), tr(ls[2]), "left")
        elif mode == 2:
            gradx, grady, gradmag = evaluate_gradient(ls[3], self.mask_right)
            edge = evaluate_edge(tr(ls[3]), tr(ls[1]), "left")
        elif mode == 3:
            gradx, grady, gradmag = evaluate_gradient(ls[4], self.mask_left_right)
            edge = (evaluate_edge(tr(ls[2]), tr(ls[4]), "left") + evaluate_edge(tr(ls[2]), tr(ls[4]), "left")) / 2
        elif mode == 4:
            gradx, grady, gradmag = evaluate_gradient(ls[mode + 1], self.mask_all)
            edge = (evaluate_edge_top(tr(ls[1]), tr(ls[5]), "top") + evaluate_edge_top(tr(ls[2]), tr(ls[5]), "right")
                    + evaluate_edge_top(tr(ls[3]), tr(ls[5]), "left") + evaluate_edge_top(tr(ls[4]), tr(ls[5]), "bottom")) / 4
        elif mode == 5:
            gradx, grady, gradmag = evaluate_gradient(ls[mode + 1], self.mask_all)
        last_content = self.frames[f][vr_oracle.PROC_ORDER[mode]]
        nan = float("nan")
        style_loss, content_loss = self.percept(last_content, ls[mode + 1]) if self.percept else (nan, nan)
        if i > 6 and not self.no_consistency_eval:
            flow_eval, cert_eval = self.load_flow_cert_eval(f, mode)
            c = cert_eval  # cert_eval:expand(3, hplus, wplus)
            if self.backward_eval:
                prev_warped_eval = vr_oracle._warp(ls[mode + 1], flow_eval)
                a, b = prev_warped_eval * c, ref.prev_last_segments[mode + 1] * c
            else:
                prev_warped_eval = vr_oracle._warp(ref.prev_last_segments[mode + 1], flow_eval)
                a, b = prev_warped_eval * c, ls[mode + 1] * c
            temporal_loss = mse(a.astype(np.float32), b.astype(np.float32))
            return [gradx, grady, gradmag, edge, style_loss, content_loss, temporal_loss], 7
        elif self.no_consistency_eval:
            return [gradx, grady, gradmag, edge, style_loss, content_loss], 6
        return [gradx, grady, gradmag, edge, style_loss, content_loss, 0], 7


class EvalVRRef(vr_oracle.VRRef):
    """VRRef whose save_image runs the evaluation hook right after it, as run_fast_neural_video calls func_eval after
    func_save_image (fast_artistic_video_core.lua:210-226).  `rows` collects (numbers, n) per face, in processing order."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.hook, self.i, self.rows = None, 0, []

    def save_image(self, mode, frame):
        res = super().save_image(mode, frame)
        self.i += 1
        if self.hook is not None:
            self.rows.append(self.hook(self.i))
        return res


def run_vr_clip_eval(ref: EvalVRRef, net, frames, flows, certs, hook_kw=None, eval_flows=None, eval_certs=None, **kw):
    """vr_oracle.run_vr_clip with func_eval after every face.  Returns (outputs, per-quantity lists as core writes them)."""
    ref.hook = VREval(ref, frames, flows if eval_flows is None else eval_flows, certs if eval_certs is None else eval_certs,
                      **(hook_kw or {}))
    outs = vr_oracle.run_vr_clip(ref, net, frames, flows, certs, **kw)
    table = []
    for numbers, n in ref.rows:
        for j in range(n):
            if j >= len(table):
                table.append([])
            table[j].append(numbers[j])
    return outs, table
