/*
 * fav.h -- C ABI of libfav_b200.so: the H100-native (sm_90a) replacement for the per-frame
 * video-style-transfer hot path of manuelruder/fast-artistic-videos (reference @ bf1d072).
 *
 * Plain C: raw DEVICE pointers (unless a parameter says "host"), sizes, element strides and a
 * cudaStream_t passed as void*.  No torch / THC / Lua types.  Every entry point returns an int
 * status (FAV_OK == 0); fav_last_error() returns a thread-local message for the last failure.
 * Nothing here allocates or frees caller tensors; kernels are enqueued on the given stream and
 * NOT synchronised (same contract as the reference: BilinearSamplerBDHW.cu:123,146-150).
 *
 * Each declaration cites the reference interface it replaces (path:line under the reference).
 * The reference-side binding a maintainer would add is shown in INTEGRATION.md; the Lua shim
 * source that registers these under the reference's names is fast-artistic-videos_b200/lua/.
 *
 * Tensor conventions (the reference's): fp32, "BDHW" = NCHW.  Optical flow in the Lua loader's
 * layout: channel 0 = dy (v), channel 1 = dx (u), pixel offsets (flowFileLoader.lua:31-32,
 * BilinearSamplerBDHW.cu:72-73).  The occlusion checker takes the .flo-native layout
 * (plane 0 = u, plane 1 = v; consistencyChecker.cpp:29-33).
 */
#ifndef FAV_H_
#define FAV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FAV_API __attribute__((visibility("default")))

/* status codes */
enum {
  FAV_OK = 0,
  FAV_ERR_INVALID = 1,         /* bad argument (the Lua asserts of BilinearSamplerBDHW.lua:26-42) */
  FAV_ERR_CUDA = 2,            /* cudaGetLastError() != success (BilinearSamplerBDHW.cu:146-150)   */
  FAV_ERR_NOT_IMPLEMENTED = 3, /* gradient entry points (BilinearSamplerBDHW.cu:171-184)           */
  FAV_ERR_IO = 4,
  FAV_ERR_UNSUPPORTED = 5,     /* arch token / device the sm_90a path does not cover              */
  FAV_ERR_NO_DEVICE = 6        /* no CUDA device: there is NO CPU fallback, calls fail loudly      */
};

/* warp border semantics */
enum {
  FAV_BORDER_PER_TAP = 0,  /* CUDA path: each out-of-range corner contributes 0
                              (BilinearSamplerBDHW.cu:92-101)                                       */
  FAV_BORDER_PAD_PIXEL = 1 /* CPU path of utils.warp_image: image.warp(...,'pad',0)
                              (fast_artistic_video/utils.lua:145-147): whole pixel = pad value when
                              the source coordinate is off-image, else clamped neighbours            */
};

FAV_API const char *fav_last_error(void);
FAV_API int fav_version(void);
/* number of kernels this library has launched in the calling process (bench.py "gpu_launches") */
FAV_API uint64_t fav_launch_count(void);
FAV_API int fav_device_count(void);

/* ---------------------------------------------------------------------------------------------
 * a-1  nn.BilinearSamplerBDHW
 * replaces cunn_BilinearSamplerBDHW_updateOutput        stnbdhw/BilinearSamplerBDHW.cu:111-152
 *      (kernel BilinearSamplerBDHW_bilinearSamplingFromGrid                         :48-109)
 * img  [B,C,Hin,Win], grid [B,2,Hout,Wout] (ch0 = dy, ch1 = dx), out [B,C,Hout,Wout];
 * *_stride are ELEMENT strides (arbitrary strides honoured, as the reference kernel does :123-142).
 * ------------------------------------------------------------------------------------------- */
FAV_API int fav_bilinear_sampler_bdhw_update_output(const float *img, const int64_t img_size[4],
                                                    const int64_t img_stride[4], const float *grid,
                                                    const int64_t grid_size[4],
                                                    const int64_t grid_stride[4], float *out,
                                                    const int64_t out_stride[4], int border_mode,
                                                    void *stream);
/* replaces cunn_BilinearSamplerBDHW_updateGradInput / _updateGradInputOnlyGrid (:171-184):
 * always FAV_ERR_NOT_IMPLEMENTED with the reference's message. */
FAV_API int fav_bilinear_sampler_bdhw_update_grad_input(void);
FAV_API int fav_bilinear_sampler_bdhw_update_grad_input_only_grid(void);

/* a-2  utils.warp_image(img, map, dtype)           fast_artistic_video/utils.lua:141-149
 * img [C,Hin,Win] contiguous, flow [2,Hout,Wout] contiguous, out [C,Hout,Wout]. */
FAV_API int fav_warp_image(const float *img, int C, int Hin, int Win, const float *flow, int Hout,
                           int Wout, float *out, int border_mode, void *stream);

/* a-5  utils.min_filter(batch, r)                  fast_artistic_video/utils.lua:161-169
 * in/out [n,H,W] contiguous: 1 - maxpool_{r x r, stride 1, pad floor(r/2)}(1 - x). r odd, <= 15. */
FAV_API int fav_min_filter(const float *in, float *out, int n, int H, int W, int r, void *stream);

/* a-6  preprocess.vgg.preprocess / deprocess       fast_artistic_video/preprocess.lua:57-62, :66-71
 * in/out [N,3,H,W] contiguous. */
FAV_API int fav_vgg_preprocess(const float *in, float *out, int N, int H, int W, void *stream);
FAV_API int fav_vgg_deprocess(const float *in, float *out, int N, int H, int W, void *stream);

/* a-8 (front half)  the 7-channel net input of run_next_image
 *                                               fast_artistic_video_core.lua:161-171
 * ONE fused kernel: warp(prev, flow) -> preprocess -> * cert -> + fill, preprocess(content), concat.
 * content, prev [3,H,W] RGB; flow [2,H,W] (dy,dx); cert [H,W]; fill [3,H,W] or NULL ('vgg-mean',
 * generate_fill :108-117); flow_mask [H,W] or NULL (:169); out7 [7,H,W]. */
FAV_API int fav_temporal_input(const float *content, const float *prev, const float *flow,
                               const float *cert, const float *fill, const float *flow_mask,
                               float *out7, int H, int W, int border_mode, void *stream);
/* The WHOLE temporal-consistency stage in one kernel (north star): certainty from the forward/backward flow pair
 * (checkConsistency, consistencyChecker.cpp:99-125, 3-argument mode) or from a given plane, utils.min_filter
 * (utils.lua:161-169), then the fused warp + preprocess + mask + concat above.  Bit-identical to fav_consistency_check ->
 * fav_min_filter -> fav_temporal_input.  flow_bw [2,H,W] (dy,dx) = (v,u) of the backward flow (drives the warp AND is
 * flow1 of the checker); exactly one of flow_fw_uv [2,H,W] (u,v) / cert_raw [H,W] is non-NULL; min_filter_r =
 * opt.occlusions_min_filter (odd, <= 15; 0/1 = none); cert_out [H,W] or NULL receives the filtered certainty.
 * Needs W % 4 == 0 and 16-byte aligned planes (FAV_ERR_UNSUPPORTED otherwise). */
FAV_API int fav_temporal_stage(const float *content, const float *prev, const float *flow_bw, const float *flow_fw_uv,
                               const float *cert_raw, const float *fill, const float *flow_mask, float *out7,
                               float *cert_out, int H, int W, int min_filter_r, int border_mode, void *stream);
/* a-9 (front half)  run_image with model_img == nil: cat(pre(img), fill(cert=0), zeros)  :133-137 */
FAV_API int fav_first_frame_input(const float *content, const float *fill, float *out7, int H, int W,
                                  void *stream);

/* f-4  temporal loss of -evaluate               fast_artistic_video.lua:128-151 (func_eval)
 * adds sum_{c,y,x} (warp(prev, flow)*cert - cur*cert)^2 to the DEVICE double *sum_dev (caller zeroes it);
 * nn.MSECriterion's value is that sum / (3*H*W).  prev, cur [3,H,W]; flow [2,H,W] (dy,dx); cert [H,W]. */
FAV_API int fav_temporal_mse(const float *prev, const float *cur, const float *flow, const float *cert, int H, int W,
                             int border_mode, double *sum_dev, void *stream);

/* ---------------------------------------------------------------------------------------------
 * a-11  checkConsistency                       consistencyChecker/consistencyChecker.cpp:80-134
 * flow1, flow2: [2,H,W] planar, plane 0 = u, plane 1 = v (readMiddlebury :16-36).
 * structure: [H,W] normalised corner measure or NULL (3-argument mode, :161-163);
 * structure_avg: CMatrix::avg of it (CMatrix.h:1245-1251), ignored when structure == NULL.
 * reliable_u8 [H,W]: the PGM payload in {0,255} (clip + (char) cast, :169-171, CMatrix.h:1068), may be NULL.
 * cert_f32   [H,W]: reliable/255 as image.load(pgm,1) yields it (fast_artistic_video.lua:103), may be NULL.
 * Evaluated with the reference's mixed float/double arithmetic: results are bit-identical.
 * ------------------------------------------------------------------------------------------- */
FAV_API int fav_consistency_check(const float *flow1, const float *flow2, const float *structure,
                                  float structure_avg, uint8_t *reliable_u8, float *cert_f32, int W,
                                  int H, void *stream);
/* a-12  computeCorners + normalize(0,1) + avg   consistencyChecker.cpp:39-78,158-159; CMatrix.h:721-736
 * image [Z,H,W] planes with values 0..255 (CTensor::readFromPPM, CTensor.h:888-936); corners [H,W];
 * workspace: device scratch of fav_compute_corners_workspace(Z,W,H) bytes; avg_out: DEVICE float. */
FAV_API size_t fav_compute_corners_workspace(int Z, int W, int H);
FAV_API int fav_compute_corners(const float *image, int Z, int W, int H, float rho, float *corners,
                                float *avg_out, void *workspace, void *stream);

/* ---------------------------------------------------------------------------------------------
 * a-V / f-4  VR (cube-map) post-processing
 * utils.median_filter(img, r)                       fast_artistic_video/utils.lua:151-159
 *   in [C,H,W] -> out [C,H-r+1,W-r+1] (valid region), lower median of the r*r window; r in {1,3,5}.
 *   (the reference casts to float on the CPU for this: "Median is not defined for CudaTensors")
 * fused 4-way border blend of one cube face         fast_artistic_video_vr.lua:146-152,454-509
 *   out = base*(1-mask) + mask * sum_i warp(rot_i(sides[i]), maps[i]) / div      (combineSides + blend)
 *   base, sides[i], out [3,S,S]; maps[i] [2,S,S] (dy,dx; sentinel 99999 outside the strip); div, mask [S,S];
 *   anti_mask [S,S] or NULL: the reference forms 1 - grad_mask_all in DOUBLE and casts it to the tensor type (:456);
 *   pass that tensor for bit parity, NULL = 1 - mask evaluated in fp32;
 *   rot[i]: 0 none, 1 rotate90, 2 rotateMinus90, 3 rotate180 (:134-144).
 * ------------------------------------------------------------------------------------------- */
FAV_API int fav_median_filter(const float *in, float *out, int C, int H, int W, int r, void *stream);
FAV_API int fav_vr_blend_sides(const float *base, const float *const sides[4], const float *const maps[4],
                               const int rot[4], const float *div, const float *mask, const float *anti_mask,
                               float *out, int S, void *stream);
/* f-4  gradient metric of the VR driver's -evaluate   evaluate_gradient, fast_artistic_video_vr.lua:344-387
 * face [3,H,W] fp32 (a stylized cube face, untrimmed), mask [H,W] fp32 (the min-filtered blend mask).  In double from the
 * fp32 values: gx = max_c |f[c][y][x+2]-f[c][y][x]| on [H,W-2], gy = max_c |f[c][y+2][x]-f[c][y][x]| on [H-2,W];
 * MX / MY = 3x3 stride-1 max-pool (padding cells ignored) of |m[y][x+2]-m[y][x]| / |m[y+2][x]-m[y][x]|.
 * OVERWRITES the DEVICE doubles sums_dev[0..5] = { sum gx, sum gy, sum MX, sum MY, sum gx*MX, sum gy*MY }; the ratios
 * gradx / grady / gradmag are formed from them by the caller.  Fixed summation order: bit-identical from call to call.
 * H, W >= 3.  Per-CTA partials come from the stream's memory pool (cudaMallocAsync) and are freed on it. */
FAV_API int fav_vr_eval_gradient(const float *face, const float *mask, int H, int W, double *sums_dev, void *stream);

/* a-3 / a-13  Middlebury .flo (HOST side)          flowFileLoader.lua:17-37, consistencyChecker.cpp:16-36
 * layout 0: [dy,dx] (Lua loader order); layout 1: [u,v] (checker order). out: host [2,H,W] with room for capacity_floats
 * floats: the header is re-validated against the file size AND the capacity (a producer may rewrite the file between
 * fav_flo_read_header and fav_flo_read: utils.wait_for_file protocol); FAV_ERR_IO, never an exception, on any mismatch. */
FAV_API int fav_flo_read_header(const char *path, int *W, int *H);
FAV_API int fav_flo_read(const char *path, float *out_host, size_t capacity_floats, int layout);
/* f-2  binary PPM (P6) / PGM (P5) -> planar fp32 [C,H,W] = byte / divisor (HOST side)
 * divisor 255: image.load(path, 3|1) (fast_artistic_video.lua:95,103); divisor 1: CTensor::readFromPPM planes 0..255
 * (consistencyChecker/CTensor.h:888-936, '#' comment lines honoured). */
FAV_API int fav_pnm_read_header(const char *path, int *W, int *H, int *C);
FAV_API int fav_pnm_read_f32(const char *path, float *out_host, size_t capacity_floats, float divisor);
/* f-2  the RAW payloads for callers that convert on the GPU (fav_session_run_frame_bytes): the P5 / P6 bytes as stored
 * (interleaved RGB; what image.load decodes, fast_artistic_video.lua:95,103) and the .flo (u,v) pairs as stored
 * (flowFileLoader.lua:28-34).  Sizes are returned and validated against the caller's capacity. */
FAV_API int fav_pnm_read_u8(const char *path, unsigned char *out_host, size_t capacity_bytes, int *W, int *H, int *C);
FAV_API int fav_flo_read_raw(const char *path, float *out_uv_pairs_host, size_t capacity_floats, int *W, int *H);

/* ---------------------------------------------------------------------------------------------
 * a-N*  the stylization network                fast_artistic_video/models_video.lua:55-140
 * fav_net_create parses the reference's arch string (tokens cXsY-Z, dX, uX, UX, RX) with
 * padding_type 'reflect-start' (train_video.lua:25; the lazily inserted SpatialReflectionPadding
 * :319-324 is part of the net), InstanceNormalization (InstanceNormalization.lua:33-53), Tanh,
 * MulConstant(tanh_constant), TotalVariation (identity fwd).  Parameters are addressed by name:
 *   "l<i>.weight|bias" conv (Torch layout: conv [Cout,Cin,k,k]; full conv [Cin,Cout,k,k]),
 *   "l<i>.n.weight|bias" IN after layer i, "l<i>.c1|c2.*", "l<i>.n1|n2.*" inside residual block i.
 * ------------------------------------------------------------------------------------------- */
typedef struct fav_net fav_net_t;

FAV_API int fav_net_create(const char *arch, const char *padding_type, float tanh_constant, int in_dim,
                           fav_net_t **out);
/* fav_net_create with the normalisation layer chosen by -use_instance_norm (train_video.lua:22): norm "instance"
 * (= fav_net_create) or "batch", nn.SpatialBatchNormalization wherever the default has InstanceNormalization
 * (models_video.lua:21-25,33-37,121-127), run in evaluate mode (fast_artistic_video_core.lua:46): y = (x - running_mean) /
 * sqrt(running_var + eps) * weight + bias.  Each norm "<n>" then has the parameters "<n>.weight|bias|running_mean|running_var"
 * [C] and "<n>.eps" [1].  fav_net_finalize folds every BN that follows a convolution into that convolution (its bias and a
 * per-channel scale) and refuses (FAV_ERR_INVALID, naming the norm) non-finite values or running_var + eps <= 0. */
FAV_API int fav_net_create_norm(const char *arch, const char *padding_type, float tanh_constant, int in_dim, const char *norm,
                                fav_net_t **out);
FAV_API void fav_net_destroy(fav_net_t *net);
FAV_API int fav_net_num_params(const fav_net_t *net);
/* name_out: >= 64 bytes; shape_out[4] (unused dims = 1); returns element count via *numel */
FAV_API int fav_net_param_info(const fav_net_t *net, int index, char *name_out, int64_t shape_out[4],
                               int64_t *numel);
FAV_API int fav_net_set_param(fav_net_t *net, const char *name, const float *host_data, int64_t numel);
/* upload + repack weights for the tensor-core path; must be called once after all set_param calls */
FAV_API int fav_net_finalize(fav_net_t *net);
/* conv implementation: 0 = tensor-core (wgmma) implicit GEMM (default), 1 = CUDA-core debug comparator.  The comparator
 * always computes in exact fp32, whatever fav_net_set_precision says. */
FAV_API int fav_net_set_conv_impl(fav_net_t *net, int impl);
/* Precision of the stylization net's tensor-core convolutions.  An addition: the reference computes in fp32 only.
 *   "pair" (default): every operand is an fp16 pair hi + lo and each K step runs three MMAs (hi*hi + lo*hi + hi*lo), fp32
 *          accumulation: fp32 parity.
 *   "fp16": single pass, one MMA per K step on the fp16 hi halves (activations rounded to fp16, weights as packed), fp32
 *          accumulation.  Faster; a deprocessed [0,1] frame moves by about one 8-bit level (DESIGN.md §2).  Not
 *          bit-comparable with "pair": a recurrent clip drifts apart from the exact one within tens of frames.
 * Anything else: FAV_ERR_INVALID.  A change drops the net's cached plans and CUDA graphs; the next call rebuilds them in the
 * new mode.  Finish every frame in flight on the net first (fav_session_sync for a session).  Neither the CUDA-core
 * comparator nor the loss network (fav_percep_*) is affected. */
FAV_API int fav_net_set_precision(fav_net_t *net, const char *mode);
/* model:forward(input)                          fast_artistic_video_core.lua:138,172
 * in7 [in_dim,H,W] device fp32 -> out3 [3,H,W] device fp32 in net space (before deprocess). */
FAV_API int fav_net_forward(fav_net_t *net, const float *in7, int H, int W, float *out3, void *stream);
/* measurement: one forward with CUDA events around every plan step (on `stream`, synchronised on return).
 * kinds: 0 pack_input, 1 convolution (all phases), 2 IN statistics, 3 IN apply; ms: device time;
 * work: algorithmic FLOPs (kind 1, logical channel counts, SURVEY.md 8d) or algorithmic bytes (others);
 * names24: max_steps x 24 chars (may be NULL). */
FAV_API int fav_net_profile(fav_net_t *net, const float *in7, int H, int W, float *out3, int max_steps, int *kinds,
                            float *ms, double *work, char *names24, int *n_out, void *stream);
/* debugging / per-layer parity: copy activation after layer `index` (post IN/ReLU) to NCHW fp32.
 * Valid after a forward at the same H,W.  out [C,Hl,Wl]; sizes returned through C/Hl/Wl. */
FAV_API int fav_net_layer_output(fav_net_t *net, int index, float *out, int *C, int *Hl, int *Wl,
                                 void *stream);

/* Batches.  The reference nets are nn modules that take N x C x H x W (InstanceNormalization.lua:33-53 normalises per (n, c);
 * train_video.lua:60 trains with -batch_size 4).  The *_batch calls take B frames of one size stored one after the other and run
 * them through one plan: every kernel covers all B images in one launch, and a run_* call is still ONE graph launch.  Image b of
 * a batch is bit-identical to the same frame run alone.  B = 1 is the single-frame call.  FAV_ERR_INVALID for B < 1, B > 64, or
 * a batch whose activation buffers would exceed the activation budget even when shared (fav_net_set_activation_budget, checked
 * before they are allocated).
 *
 * model:forward(input) of a batch                fast_artistic_video_core.lua:138,172
 * in [B,in_dim,H,W] device fp32 -> out3 [B,3,H,W] device fp32 in net space. */
FAV_API int fav_net_forward_batch(fav_net_t *net, const float *in, int B, int H, int W, float *out3, void *stream);
/* fav_net_layer_output for image b of the last forward's batch (models_video.lua:55-140 layer `index`), computed with the
 * style that forward gave image b (fav_net_set_batch_styles). */
FAV_API int fav_net_layer_output_image(fav_net_t *net, int index, int b, float *out, int *C, int *Hl, int *Wl, void *stream);

/* Style banks.  An addition: the reference loads one model per run (fast_artistic_video_core.lua:39-47), and every released
 * video model (candy, mosaic, ...) has the same architecture (models_video.lua:55-140).  A finalized net can hold S >= 1
 * weight sets of its own architecture, its styles; style 0 is its own parameters.  A batch may then give each image its own
 * style: image b of a *_batch call (or fav_net_forward_batch) is bit-identical to the same frame run alone on the net that
 * style came from.
 *
 * fav_net_add_style: style S = src's parameters (its style 0), copied into the net: src may be destroyed afterwards.  Both
 * nets must be finalized and agree on arch, padding_type, tanh_constant, in_dim and norm (fast_artistic_video_core.lua:39-47
 * loads them with the checkpoint); otherwise FAV_ERR_INVALID naming the first property that differs.  At most 64 styles (the
 * batch limit).  *index_out = S.  Drops the net's cached plans and CUDA graphs, as fav_net_set_precision does. */
FAV_API int fav_net_add_style(fav_net_t *net, const fav_net_t *src, int *index_out);
/* The number of styles the net holds (1 until fav_net_add_style).  models_video.lua:55-140 builds one. */
FAV_API int fav_net_num_styles(const fav_net_t *net);
/* The style of each image of later calls (fast_artistic_video_core.lua:121-180 run_image / run_next_image, batched): image b
 * runs style styles[b].  n == 0 restores the default, style 0 for every image.  With n > 0 every later forward or run_* call
 * must have B == n, and each entry must lie in [0, S); otherwise FAV_ERR_INVALID.  A change rebuilds no plan and re-captures
 * no graph: each call writes the assignment on its own stream before its kernels. */
FAV_API int fav_net_set_batch_styles(fav_net_t *net, const int *styles, int n);

/* Activation memory.  A plan (one per batch size B and frame size H x W, built at its first call) gives every activation its
 * own buffer when their total fits the net's activation budget.  When it does not, activations whose lifetimes do not overlap
 * share one arena, and the kernels and their order stay the same: the output is bit-identical to the all-live plan's.  On
 * such a plan fav_net_layer_output returns FAV_ERR_INVALID for a layer whose activation a later layer has taken over (the
 * input of the final layer stays readable).  A plan whose shared arena exceeds the budget as well is refused with
 * FAV_ERR_INVALID, both figures in the message.
 *
 * The budget applies to plans created after the call; plans already built keep their buffers.  Default: 32 GiB. */
FAV_API int fav_net_set_activation_budget(fav_net_t *net, size_t bytes);
/* The activation bytes a (B, H, W) plan takes with every activation in its own buffer (*all_live) and with buffers shared by
 * lifetime (*shared), without allocating anything.  After fav_net_finalize. */
FAV_API int fav_net_plan_bytes(fav_net_t *net, int B, int H, int W, size_t *all_live, size_t *shared);

/* ---------------------------------------------------------------------------------------------
 * f-5  the perceptual loss network of -evaluate: nn.PerceptualCriterion with nn.ContentLoss / nn.StyleLoss
 *      (fast_artistic_video/PerceptualCriterion.lua:27-155, ContentLoss.lua:39-48, StyleLoss.lua:39-55,
 *      GramMatrix.lua:31-53), set up as fast_artistic_video_core.lua:74-98 does.
 * The loss network is a chain of modules, 8 ints each (module i of the file's nn.Sequential is entry i-1):
 *   {0, nInputPlane, nOutputPlane, k, stride, pad, 0, 0}  SpatialConvolution (square kernel)
 *   {1, 0, ...}                                            ReLU
 *   {2, kW, kH, dW, dH, padW, padH, ceil_mode}             SpatialMaxPooling
 * Layer indices are 1-based top-level module indices; the module's OUTPUT is the feature map (conv + bias, ReLU output,
 * pooled map).  Modules after the deepest loss layer are dropped (layer_utils.lua:146-165).  agg_type: 0 'gram', 1 'mean'
 * (-style_target_type, StyleLoss.lua:14-24).  FAV_ERR_UNSUPPORTED names the module of a geometry the tensor-core path does
 * not run.
 * ------------------------------------------------------------------------------------------- */
typedef struct fav_percep fav_percep_t;
FAV_API int fav_percep_create(int n_modules, const int *modules8, int n_content, const int *content_layers,
                              const double *content_weights, int n_style, const int *style_layers,
                              const double *style_weights, int agg_type, fav_percep_t **out);
FAV_API void fav_percep_destroy(fav_percep_t *p);
/* weights of convolution module `module_index` (1-based): host fp32 [nOutputPlane, nInputPlane, k, k] and [nOutputPlane] */
FAV_API int fav_percep_set_conv(fav_percep_t *p, int module_index, const float *weight, int64_t weight_numel,
                                const float *bias, int64_t bias_numel);
FAV_API int fav_percep_finalize(fav_percep_t *p);
/* percep_crit:setStyleTarget(preprocess(style_image))      fast_artistic_video_core.lua:93-97, PerceptualCriterion.lua:72-80
 * rgb [3,H,W] device fp32 in [0,1] (already scaled to -style_image_size by the caller); the VGG preprocess runs on the GPU. */
FAV_API int fav_percep_set_style_target(fav_percep_t *p, const float *rgb, int H, int W, void *stream);
/* evaluate_image(content, stylized)                        fast_artistic_video_core.lua:101-106
 * content, stylized [3,H,W] device fp32 RGB [0,1] (stylized: the unclamped frame); returns total_content_loss and
 * total_style_loss through HOST doubles (synchronises `stream`).  FAV_ERR_UNSUPPORTED if an activation left the fp16 operand
 * range (|x| > 65504): the losses are then not computed from clamped values. */
FAV_API int fav_percep_evaluate(fav_percep_t *p, const float *content, const float *stylized, int H, int W,
                                double *content_loss, double *style_loss, void *stream);
/* tests: feature map of loss layer `index` from the last forward, fp32 NCHW [C,Hl,Wl] (out may be NULL for the sizes).
 * pass 0: the content-target forward of the last evaluation (content layers only); pass 1: the evaluated image, or the style
 * image after fav_percep_set_style_target (PerceptualCriterion.lua:85-93,117-125). */
FAV_API int fav_percep_layer_output(fav_percep_t *p, int pass, int index, float *out, int *C, int *Hl, int *Wl,
                                    void *stream);
/* tests: the aggregate (StyleLoss.lua:40-43) of style layer k (0-based position in the style layer list) as DEVICE
 * doubles: Gram matrix C*C (GramMatrix.lua:31-53) or C means; which 0 = style target, 1 = last evaluated image. */
/* tests: the fp32 output (bias included, before any ReLU or pooling) of convolution module `module_index` from the last
 * fav_percep_forward_backward, fp32 NCHW [C,H,W] (out may be NULL for the sizes): the values whose ReLU masks (> 0) and
 * max-pooling arg-maxes the backward pass used.  FAV_ERR_INVALID if the last call was an evaluation or a style target (those
 * share one buffer between convolutions) or the module is not a convolution. */
FAV_API int fav_percep_conv_output(fav_percep_t *p, int module_index, float *out, int *C, int *H, int *W, void *stream);
FAV_API int fav_percep_style_stat(fav_percep_t *p, int which, int k, double *out, int *n, void *stream);
/* percep_crit:forward(input, {content_target=...}) then percep_crit:backward(input, target)   train_video.lua:343-345,
 * PerceptualCriterion.lua:117-161, ContentLoss.lua:50-59, StyleLoss.lua:57-67, GramMatrix.lua:54-78.
 * content_pre, input_pre [3,H,W] device fp32 in NET space (BGR, 255 x - mean; content_pre may be NULL without content layers);
 * writes grad_input [3,H,W] (d total / d input_pre), the two totals and, if layer_losses is not NULL, strength * MSE of every
 * loss layer (content layers, then style layers) through HOST doubles (synchronises `stream`).  FAV_ERR_UNSUPPORTED names the
 * module, before any kernel launch, unless every convolution up to the deepest loss layer
 *  - is stride 1 with pad (k-1)/2, and
 *  - has an input gradient (a nOutputPlane -> nInputPlane convolution) the tensor-core planner runs: nOutputPlane <= 8, or
 *    nOutputPlane rounded up to 8 is an even number of 8-channel blocks (16, 32, 48, ...) that splits into at most 16 K groups
 *    (blocks of 4 when the count is a multiple of 4, else of 2; a 5x5 or 7x7 filter over groups of 4 blocks, and a 7x7 over
 *    groups of 2, takes a group per filter row).  Between convolutions only the deepest convolution's nOutputPlane is free, so e.g. 17, 33, 100, 130 or 200 there is
 *    refused;
 * and no convolution is followed by more than 7 loss layers before the next one (8 after the deepest).  The first call at a
 * size keeps every convolution's fp32 output (about 1.1 GB at 1280x720 to relu4_3). */
FAV_API int fav_percep_forward_backward(fav_percep_t *p, const float *content_pre, const float *input_pre, int H, int W,
                                        float *grad_input, double *content_loss, double *style_loss, double *layer_losses,
                                        void *stream);
/* pixel_crit:forward / backward(out2 .* cert, out1_warped_masked)   train_video.lua:117-126,354-366
 * out2, prev_warped_masked [N,3,H,W], cert [N,1,H,W] device fp32; type 0 L2 (MSECriterion), 1 L1 (AbsCriterion), 2 SmoothL1;
 * sizeAverage.  grad_accum [N,3,H,W] += weight * d loss / d (out2 .* cert) -- NOT multiplied by cert, as train_video.lua:357-364
 * adds it; *loss = weight * loss (HOST double, synchronises `stream`). */
FAV_API int fav_pixel_loss_grad(const float *out2, const float *prev_warped_masked, const float *cert, int N, int H, int W,
                                int type, float weight, float *grad_accum, double *loss, void *stream);
/* nn.TotalVariation:updateGradInput with gradOutput = grad_accum   TotalVariation.lua:19-35
 * x, grad_accum [N,3,H,W] device fp32: grad_accum += strength * (TV gradient over the {1,-2} ranges). */
FAV_API int fav_tv_grad(const float *x, int N, int H, int W, float strength, float *grad_accum, void *stream);

/* diagnostics: per-CTA timeline of the following tensor-core convolution launches (entry / set-up /
 * exit clock64 marks, 64 u64 words per CTA, launches appended) into a caller-owned DEVICE buffer; NULL = off. */
FAV_API int fav_debug_set_trace(void *dev_buf, size_t bytes);
FAV_API size_t fav_debug_trace_words(void);

/* a-9  run_image                               fast_artistic_video_core.lua:121-158
 * content [3,H,W] RGB [0,1] -> out_rgb [3,H,W] = deprocess(model(...))[1].  A net created with in_dim = 7 is the video model
 * fed cat(pre(img), fill, zeros) (model_img == nil, :133-138); in_dim = 3 is a separate image model fed pre(img) (:146, fill
 * is ignored).  -scale_factor != 1 is fav_run_image_scaled below.
 * fav_run_image / fav_run_next_image enqueue the fused input kernel plus ONE CUDA-graph launch of the network (captured on
 * the second call for each distinct out_rgb pointer, 8 graphs cached per frame size): ping-pong a few output buffers.
 * One stream at a time per net (it owns the activation buffers), like model:forward in the reference. */
FAV_API int fav_run_image(fav_net_t *net, const float *content, const float *fill, int H, int W,
                          float *out_rgb, void *stream);
/* a-9 with -scale_factor                        fast_artistic_video_core.lua:121-158 (fast_artistic_video.lua:42)
 * content [3,H,W] -> out_rgb [3,H,W] = image.scale(deprocess(model_img(pre(image.scale(content, W*sf, H*sf, 'bicubic')))),
 * W, H, 'bicubic') (:127-130,146-152), unclamped (the reference keeps it as last_frame_stylized, fast_artistic_video.lua:169).
 * scale_factor == 1 is exactly fav_run_image(net, content, NULL, H, W, out_rgb, stream).  Otherwise the net must be an image
 * model (in_dim 3): the video model's input would join the scaled frame with an unscaled fill, which the reference's torch.cat
 * refuses (:133-138).  h = H*sf and w = W*sf (in double) must be integers, and h x w must satisfy the frame rules of every
 * run_* call (multiples of 4, at least 16, larger than the reflection padding).  Every refusal is FAV_ERR_INVALID, before any
 * device work.  The network runs at h x w as ONE cached graph launch, between the two fav_image_scale_bicubic kernels. */
FAV_API int fav_run_image_scaled(fav_net_t *net, const float *content, int H, int W, double scale_factor, float *out_rgb,
                                 void *stream);
/* image.scale(src, Wout, Hout, 'bicubic') of the `image` rock (fast_artistic_video_core.lua:128,151; the rock is not vendored,
 * DESIGN.md 8 states the reading): in [C,Hin,Win] -> out [C,Hout,Wout], planar fp32.  Separable Catmull-Rom on an
 * align-corners grid, linearly extrapolated borders, no prefilter, no clamping; a side of equal size is copied.  Sizes 2 to
 * 65535 (FAV_ERR_INVALID otherwise, a side of 1 included). */
FAV_API int fav_image_scale_bicubic(const float *in, float *out, int C, int Hin, int Win, int Hout, int Wout, void *stream);
/* a-8  run_next_image                           fast_artistic_video_core.lua:161-180
 * (+ func_make_last_frame_warped, fast_artistic_video.lua:153-158: the warp of prev_rgb by flow) */
FAV_API int fav_run_next_image(fav_net_t *net, const float *content, const float *prev_rgb,
                               const float *flow, const float *cert, const float *fill,
                               const float *flow_mask, int H, int W, int border_mode, float *out_rgb,
                               void *stream);

/* a-8 including func_load_cert + utils.min_filter (core.lua:206-208): ONE temporal-stage kernel (fav_temporal_stage, writing
 * the network's first operand directly) + one graph launch.  Arguments as fav_temporal_stage; falls back to the three
 * separate kernels when the vector path does not apply. */
FAV_API int fav_run_next_image_flows(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow_bw,
                                     const float *flow_fw_uv, const float *cert_raw, const float *fill,
                                     const float *flow_mask, int H, int W, int min_filter_r, int border_mode,
                                     float *out_rgb, void *stream);
/* fav_run_next_image_flows with the certainty in the 4-argument mode of the stylization scripts (makeOptFlow_deepflow.sh:58-60;
 * consistencyChecker.cpp:39-78,122-124,154-160; read as reliable_[i]_{i-1}.pgm by fast_artistic_video.lua:99-112): the
 * structure term comes from `content` (byte/255 planes of frame i, the image of the checker's call), flow_bw = [dy,dx] of
 * backward_i_{i-1}.flo, flow_fw_uv = forward_{i-1}_i.flo in (u,v) order.  The corners, their exact average and the fused
 * stage run on the device.  One image; H, W >= 3. */
FAV_API int fav_run_next_image_flows_structure(fav_net_t *net, const float *content, const float *prev_rgb,
                                               const float *flow_bw, const float *flow_fw_uv, const float *fill,
                                               const float *flow_mask, int H, int W, int min_filter_r, int border_mode,
                                               float *out_rgb, void *stream);

/* Batched frame calls (see fav_net_forward_batch): every plane argument holds B images one after the other -- content,
 * prev_rgb, fill, out_rgb [B,3,H,W]; flow, flow_bw, flow_fw_uv [B,2,H,W]; cert, cert_raw, flow_mask [B,H,W].  Each image keeps
 * its own recurrent state (the caller's prev_rgb[b]), so B independent clips advance one frame per call.
 *   run_image                                    fast_artistic_video_core.lua:121-158 */
FAV_API int fav_run_image_batch(fav_net_t *net, const float *content, const float *fill, int B, int H, int W, float *out_rgb,
                                void *stream);
/*   run_next_image                               fast_artistic_video_core.lua:161-180 */
FAV_API int fav_run_next_image_batch(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow,
                                     const float *cert, const float *fill, const float *flow_mask, int B, int H, int W,
                                     int border_mode, float *out_rgb, void *stream);
/*   run_next_image with func_load_cert + utils.min_filter inside (core.lua:206-208) */
FAV_API int fav_run_next_image_flows_batch(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow_bw,
                                           const float *flow_fw_uv, const float *cert_raw, const float *fill,
                                           const float *flow_mask, int B, int H, int W, int min_filter_r, int border_mode,
                                           float *out_rgb, void *stream);

/* ---------------------------------------------------------------------------------------------
 * a-10  frame loop with HOST buffers (the reference-facing call bench.py's e2e times)
 *                                               fast_artistic_video_core.lua:189-229
 * A session owns device + pinned staging buffers for one H x W stream on one GPU, keeps the
 * recurrent state last_frame_stylized on the device as unclamped fp32 (fast_artistic_video.lua:169)
 * and overlaps H2D / compute / D2H on three streams.
 * ------------------------------------------------------------------------------------------- */
typedef struct fav_session fav_session_t;
FAV_API int fav_session_create(fav_net_t *net, int H, int W, fav_session_t **out);
FAV_API void fav_session_destroy(fav_session_t *s);
/* -model_img (fast_artistic_video.lua:24, core.lua:61-68,146): single images go through this 3-channel image model instead
 * of the video model with an empty prior; NULL = "self".  The session does not own it. */
FAV_API int fav_session_set_image_model(fav_session_t *s, fav_net_t *net_img);
/* frame 1 (func_is_single_image): host content [3,H,W] fp32 -> host out [3,H,W] fp32 */
FAV_API int fav_session_run_image(fav_session_t *s, const float *content_host, float *out_host);
/* frames >= 2: host content, host flow [2,H,W] (dy,dx), host cert [H,W] fp32 in [0,1] BEFORE the
 * min filter (func_load_cert output); min_filter_r = opt.occlusions_min_filter (0 = skip). */
FAV_API int fav_session_run_next_image(fav_session_t *s, const float *content_host,
                                       const float *flow_host, const float *cert_host,
                                       int min_filter_r, int border_mode, float *out_host);
/* same, but the certainty is computed on the GPU from the forward/backward flow pair
 * (fused consistency check, 3-argument mode): flow_bw/flow_fw host [2,H,W] in .flo (u,v) order. */
FAV_API int fav_session_run_next_image_flows(fav_session_t *s, const float *content_host,
                                             const float *flow_bw_uv_host,
                                             const float *flow_fw_uv_host, int min_filter_r,
                                             int border_mode, float *out_host);
/* same in the checker's 4-argument mode, the structure term from the frame itself (fav_run_next_image_flows_structure;
 * makeOptFlow_deepflow.sh:58-60, consistencyChecker.cpp:39-78,122-124,154-160). */
FAV_API int fav_session_run_next_image_flows_structure(fav_session_t *s, const float *content_host,
                                                       const float *flow_bw_uv_host, const float *flow_fw_uv_host,
                                                       int min_filter_r, int border_mode, float *out_host);
/* completion of ONE frame: call number frame_index (0-based) of fav_session_run_* on this session has landed in its out_host
 * buffer (wait != 0 blocks; wait == 0 polls: FAV_OK / FAV_ERR_INVALID "still in flight").  Lets encoder threads consume
 * frames while later ones are still being enqueued (file-driven pipeline, fav_b200/video.py). */
FAV_API int fav_session_frame_done(fav_session_t *s, uint64_t frame_index, int wait);
/* f-2  image.save of an already quantised 8-bit image (fast_artistic_video.lua:161, fast_artistic_video_vr.lua:541-556):
 * pixels = H x W x C bytes (C = 3 RGB | 1 gray, interleaved) -> PNG (Sub filter; png_level 0 stored, 1 zlib level 1 + Z_RLE,
 * >= 2 that zlib level), deflated in nthreads concurrent bands.  HOST side. */
FAV_API int fav_png_write(const char *path, const unsigned char *pixels, int W, int H, int C, int png_level, int nthreads);
/* f-2 / (e)  the conversions of image.load / flowFile.load / func_load_cert / image.save (fast_artistic_video.lua:95-110,161;
 * flowFileLoader.lua:28-34) on DEVICE buffers: rgb_hwc H*W*3 bytes -> content [3,H,W] = byte / 255; flo_uv H*W (u,v) pairs ->
 * flow [2,H,W] = (dy,dx); cert8 H*W bytes -> cert [H,W] = byte / 255 (1 - that with invert_occlusion); and a stylized frame
 * [3,H,W] -> H*(1+3W) bytes of Sub-filtered PNG scanlines quantised like image.save.  flo_uv/flow and cert8/cert may be NULL. */
FAV_API int fav_bytes_to_planes(const unsigned char *rgb_hwc, const float *flo_uv, const unsigned char *cert8, int invert_occlusion,
                                float *content, float *flow, float *cert, int H, int W, void *stream);
FAV_API int fav_planes_to_png_rows(const float *rgb_planes, unsigned char *rows, int H, int W, void *stream);
/* f-2  one frame from FILE PAYLOADS (what image.load / flowFile.load / func_load_cert / image.save do on the host,
 * fast_artistic_video.lua:95-110,161): rgb_hwc = P6 payload (H*W*3 bytes), flo_uv = .flo payload (H*W (u,v) pairs),
 * cert8 = P5 payload of the certainty (both NULL for the first frame); png_rows_host receives H*(1+3W) bytes = the stylized
 * frame quantised like image.save as Sub-filtered PNG scanlines (ready for deflate).  Byte <-> float conversions run on the
 * GPU behind the copies (same fp32 operations as the host readers: results are bit-identical); the compute stream runs exactly
 * what fav_session_run_next_image runs.  Completion: fav_session_frame_done. */
FAV_API int fav_session_run_frame_bytes(fav_session_t *s, const unsigned char *rgb_hwc, const float *flo_uv,
                                        const unsigned char *cert8, int invert_occlusion, int min_filter_r, int border_mode,
                                        unsigned char *png_rows_host);
/* the same with both .flo payloads and no PGM: flo_bw_uv = backward_i_{i-1}.flo, flo_fw_uv = forward_{i-1}_i.flo (both NULL for
 * the first frame); the certainty is the checker's 4-argument mode with frame i as the image, computed on the GPU as
 * fav_session_run_next_image_flows_structure does (makeOptFlow_deepflow.sh:58-60, consistencyChecker.cpp:39-78,122-124,154-160). */
FAV_API int fav_session_run_frame_bytes_flows(fav_session_t *s, const unsigned char *rgb_hwc, const float *flo_bw_uv,
                                              const float *flo_fw_uv, int min_filter_r, int border_mode,
                                              unsigned char *png_rows_host);
/* f-2  the file-driven frame loop (fast_artistic_video.lua:93-170) as a native pipeline around this session: decoder threads
 * (frame PPM, certainty PGM, .flo -> pinned ring slots; [fmt]/{fmt} patterns :70-77; wait-for-file protocol utils.lua:74-80),
 * the calling thread enqueues frames, encoder threads wait per frame and write "<output_prefix>-%05d.png" (:161; zlib level
 * png_level, pixels identical to the synchronous driver's files).  Frames i = 1.. until num_frames or the first missing frame
 * file.  Blocks until the last PNG is written; frames_done / seconds may be NULL. */
FAV_API int fav_video_pipeline_run(fav_session_t *s, int H, int W, const char *input_pattern, const char *flow_pattern,
                                   const char *occlusions_pattern, const char *output_prefix, int num_frames, int min_filter_r,
                                   int invert_occlusion, int n_decode, int n_encode, int depth, int png_level, int *frames_done,
                                   double *seconds);
/* fav_video_pipeline_run without certainty PGMs: the decoder threads read the backward flow (flow_pattern) and the forward flow
 * (flow_fw_pattern, e.g. "forward_{%d}_[%d].flo"), waiting for the forward flow first as makeOptFlow_deepflow.sh:58 does, and
 * each frame runs fav_session_run_frame_bytes_flows (the checker's 4-argument mode on the GPU). */
FAV_API int fav_video_pipeline_run_flows(fav_session_t *s, int H, int W, const char *input_pattern, const char *flow_pattern,
                                         const char *flow_fw_pattern, const char *output_prefix, int num_frames, int min_filter_r,
                                         int n_decode, int n_encode, int depth, int png_level, int *frames_done, double *seconds);
/* block until every queued frame has landed in its out_host buffer */
FAV_API int fav_session_sync(fav_session_t *s);
/* device time (ms, CUDA events on the compute stream) of the last frame's GPU work */
FAV_API float fav_session_last_gpu_ms(fav_session_t *s);

#ifdef __cplusplus
}
#endif
#endif /* FAV_H_ */
