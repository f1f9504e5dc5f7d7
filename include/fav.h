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
FAV_API void fav_net_destroy(fav_net_t *net);
FAV_API int fav_net_num_params(const fav_net_t *net);
/* name_out: >= 64 bytes; shape_out[4] (unused dims = 1); returns element count via *numel */
FAV_API int fav_net_param_info(const fav_net_t *net, int index, char *name_out, int64_t shape_out[4],
                               int64_t *numel);
FAV_API int fav_net_set_param(fav_net_t *net, const char *name, const float *host_data, int64_t numel);
/* upload + repack weights for the tensor-core path; must be called once after all set_param calls */
FAV_API int fav_net_finalize(fav_net_t *net);
/* conv implementation: 0 = tensor-core (wgmma) implicit GEMM (default), 1 = CUDA-core debug comparator */
FAV_API int fav_net_set_conv_impl(fav_net_t *net, int impl);
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

/* diagnostics: per-CTA timeline of the following tensor-core convolution launches (entry / set-up /
 * exit clock64 marks, 64 u64 words per CTA, launches appended) into a caller-owned DEVICE buffer; NULL = off. */
FAV_API int fav_debug_set_trace(void *dev_buf, size_t bytes);
FAV_API size_t fav_debug_trace_words(void);

/* a-9  run_image                               fast_artistic_video_core.lua:121-158
 * content [3,H,W] RGB [0,1] -> out_rgb [3,H,W] = deprocess(model(...))[1].  A net created with in_dim = 7 is the video model
 * fed cat(pre(img), fill, zeros) (model_img == nil, :133-138); in_dim = 3 is a separate image model fed pre(img) (:146, fill
 * is ignored).  -scale_factor != 1 (bicubic image.scale of the un-vendored `image` rock, :127-129,150-152) is not built.
 * fav_run_image / fav_run_next_image enqueue the fused input kernel plus ONE CUDA-graph launch of the network (captured on
 * the second call for each distinct out_rgb pointer, 8 graphs cached per frame size): ping-pong a few output buffers.
 * One stream at a time per net (it owns the activation buffers), like model:forward in the reference. */
FAV_API int fav_run_image(fav_net_t *net, const float *content, const float *fill, int H, int W,
                          float *out_rgb, void *stream);
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
/* f-2  the file-driven frame loop (fast_artistic_video.lua:93-170) as a native pipeline around this session: decoder threads
 * (frame PPM, certainty PGM, .flo -> pinned ring slots; [fmt]/{fmt} patterns :70-77; wait-for-file protocol utils.lua:74-80),
 * the calling thread enqueues frames, encoder threads wait per frame and write "<output_prefix>-%05d.png" (:161; zlib level
 * png_level, pixels identical to the synchronous driver's files).  Frames i = 1.. until num_frames or the first missing frame
 * file.  Blocks until the last PNG is written; frames_done / seconds may be NULL. */
FAV_API int fav_video_pipeline_run(fav_session_t *s, int H, int W, const char *input_pattern, const char *flow_pattern,
                                   const char *occlusions_pattern, const char *output_prefix, int num_frames, int min_filter_r,
                                   int invert_occlusion, int n_decode, int n_encode, int depth, int png_level, int *frames_done,
                                   double *seconds);
/* block until every queued frame has landed in its out_host buffer */
FAV_API int fav_session_sync(fav_session_t *s);
/* device time (ms, CUDA events on the compute stream) of the last frame's GPU work */
FAV_API float fav_session_last_gpu_ms(fav_session_t *s);

#ifdef __cplusplus
}
#endif
#endif /* FAV_H_ */
