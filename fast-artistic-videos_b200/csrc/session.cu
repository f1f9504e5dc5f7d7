// session.cu -- a-10: the frame loop with HOST buffers (fast_artistic_video_core.lua:189-229 +
// fast_artistic_video.lua:93-170).  One session = one H x W stream on one GPU.
//
// The recurrent state last_frame_stylized stays on the device as unclamped fp32 (fast_artistic_video.lua:169).
// Three streams: H2D (frame i+1 inputs), compute (frame i), D2H (frame i-1 result); inputs and outputs are
// double buffered and ordered with events, so copies overlap compute whenever the caller's host buffers are
// pinned.  Nothing in the loop synchronises the host except fav_session_sync(); host buffers handed to a call must stay
// untouched until then (the copies are asynchronous).  Per frame the compute stream runs TWO launches: the fused
// temporal-stage kernel (fav_run_next_image_flows) and the CUDA graph of the network; the 4-argument variants run the
// corners chain of fav_compute_corners (structure tensor, transposes, IIRs, eigenvalues, normalize scan, the three kernels
// of the exact average) before them.
// The flows variant evaluates checkConsistency in its 3-argument mode (video_dataset/make_occlusions.sh:31-36); the
// flows_structure variant in the 4-argument mode of makeOptFlow_deepflow.sh:58-60, with the structure term from the frame
// being stylized: it adds the corners chain (fav_compute_corners' kernels) before the stage kernel.
#include <memory>
#include <vector>

#include "fav_common.cuh"


using namespace fav;

struct fav_session {
  fav_net_t *net = nullptr;
  fav_net_t *net_img = nullptr;  // optional separate image model for single images (-model_img, core.lua:61-68,146)
  int H = 0, W = 0;
  cudaStream_t s_h2d = nullptr, s_comp = nullptr, s_d2h = nullptr;
  struct InSet {
    float *content = nullptr, *flow = nullptr, *flow_fw = nullptr, *cert_raw = nullptr, *cert = nullptr;
    unsigned char *rgb8 = nullptr, *cert8 = nullptr;  // file payloads (fav_session_run_frame_bytes), allocated on first use
    float *flo_uv = nullptr, *flo_fw_uv = nullptr;
    cudaEvent_t uploaded = nullptr, consumed = nullptr;
    bool used = false;
  } in[2];
  float *out[2] = {nullptr, nullptr};
  unsigned char *rows8[2] = {nullptr, nullptr};  // Sub-filtered PNG scanlines of out[i] (fav_session_run_frame_bytes)
  cudaEvent_t computed[2] = {nullptr, nullptr}, downloaded[2] = {nullptr, nullptr};
  static constexpr int kDoneRing = 64;  // per-frame completion events for host threads (fav_session_frame_done)
  cudaEvent_t done[kDoneRing] = {};
  bool out_used[2] = {false, false};
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  uint64_t frame = 0;
  bool have_prev = false;
  std::vector<void *> allocs;
};

static int s_alloc(fav_session *s, float **p, size_t n) {
  void *d = nullptr;
  FAV_TRY(check_cuda(cudaMalloc(&d, n * sizeof(float)), "cudaMalloc(session)"));
  s->allocs.push_back(d);
  *p = (float *)d;
  return FAV_OK;
}

namespace {
// ---- file payloads <-> planes (f-2): what image.load / flowFile.load / image.save do on the host in the reference
// (fast_artistic_video.lua:95,103,161; flowFileLoader.lua:28-34), moved behind the copy engines.  Same fp32 operations as the
// host readers of flo_io.cpp and the quantisation of video_pipeline.cu, so files and frames are bit-identical either way.
// flo_fw (may be NULL): a forward-flow payload, written as the (u, v) planes the occlusion test reads
__global__ void __launch_bounds__(256) decode_bytes_kernel(const unsigned char *__restrict__ rgb, const float2 *__restrict__ flo,
                                                           const unsigned char *__restrict__ cert8, int invert,
                                                           float *__restrict__ content, float *__restrict__ flow,
                                                           float *__restrict__ cert, int64_t HW,
                                                           const float2 *__restrict__ flo_fw, float *__restrict__ flow_fw) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= HW) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) content[c * HW + i] = __fdiv_rn((float)rgb[3 * i + c], 255.0f);  // image.load: byte / 255
  if (flo) {
    const float2 f = __ldg(flo + i);  // .flo payload: (u, v) pairs; the loader returns [dy = v, dx = u] (flowFileLoader.lua:31-32)
    flow[i] = f.y; flow[HW + i] = f.x;
  }
  if (flo_fw) {
    const float2 f = __ldg(flo_fw + i);
    flow_fw[i] = f.x; flow_fw[HW + i] = f.y;
  }
  if (cert8) {
    float c = __fdiv_rn((float)cert8[i], 255.0f);
    if (invert) c = __fsub_rn(1.0f, c);  // -invert_occlusion (fast_artistic_video.lua:105-107)
    cert[i] = c;
  }
}

__device__ __forceinline__ int quantize_u8(float v) {  // image.save: clamp to [0,1], x255, round
  v = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
  v = floorf(__fadd_rn(__fmul_rn(v, 255.0f), 0.5f));
  return (int)(v < 0.f ? 0.f : (v > 255.f ? 255.f : v));
}

// rows: H x (1 + 3W) bytes = PNG scanlines, filter type 1 (Sub) -- ready for deflate
__global__ void __launch_bounds__(256) encode_rows_kernel(const float *__restrict__ out, unsigned char *__restrict__ rows, int H, int W) {
  const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const int64_t HW = (int64_t)H * W;
  unsigned char *dst = rows + (int64_t)y * (1 + 3 * (int64_t)W);
  if (x == 0) dst[0] = 1;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float *src = out + c * HW + (int64_t)y * W;
    const int q = quantize_u8(src[x]), pq = x > 0 ? quantize_u8(src[x - 1]) : 0;
    dst[1 + 3 * x + c] = (unsigned char)(q - pq);
  }
}
}  // namespace

extern "C" {

void fav_session_destroy(fav_session_t *s) {
  if (!s) return;
  cudaDeviceSynchronize();
  for (void *p : s->allocs) cudaFree(p);
  for (int i = 0; i < 2; ++i) {
    if (s->in[i].uploaded) cudaEventDestroy(s->in[i].uploaded);
    if (s->in[i].consumed) cudaEventDestroy(s->in[i].consumed);
    if (s->computed[i]) cudaEventDestroy(s->computed[i]);
    if (s->downloaded[i]) cudaEventDestroy(s->downloaded[i]);
  }
  for (cudaEvent_t e : s->done)
    if (e) cudaEventDestroy(e);
  if (s->t0) cudaEventDestroy(s->t0);
  if (s->t1) cudaEventDestroy(s->t1);
  if (s->s_h2d) cudaStreamDestroy(s->s_h2d);
  if (s->s_comp) cudaStreamDestroy(s->s_comp);
  if (s->s_d2h) cudaStreamDestroy(s->s_d2h);
  delete s;
}

int fav_session_create(fav_net_t *net, int H, int W, fav_session_t **out) {
  FAV_REQUIRE(net && out, "fav_session_create: null argument");
  FAV_REQUIRE(H >= 16 && W >= 16 && H % 4 == 0 && W % 4 == 0,
              "fav_session_create: frame size %dx%d: H and W must be multiples of 4 and >= 16 (reflect-start nets restore the "
              "input size only then)", W, H);
  FAV_TRY(require_device());
  std::unique_ptr<fav_session, void (*)(fav_session *)> s(new fav_session(), fav_session_destroy);
  s->net = net; s->H = H; s->W = W;
  FAV_TRY(check_cuda(cudaStreamCreateWithFlags(&s->s_h2d, cudaStreamNonBlocking), "cudaStreamCreate"));
  FAV_TRY(check_cuda(cudaStreamCreateWithFlags(&s->s_comp, cudaStreamNonBlocking), "cudaStreamCreate"));
  FAV_TRY(check_cuda(cudaStreamCreateWithFlags(&s->s_d2h, cudaStreamNonBlocking), "cudaStreamCreate"));
  const size_t HW = (size_t)H * W;
  for (int i = 0; i < 2; ++i) {
    FAV_TRY(s_alloc(s.get(), &s->in[i].content, 3 * HW));
    FAV_TRY(s_alloc(s.get(), &s->in[i].flow, 2 * HW));
    FAV_TRY(s_alloc(s.get(), &s->in[i].flow_fw, 2 * HW));
    FAV_TRY(s_alloc(s.get(), &s->in[i].cert_raw, HW));
    FAV_TRY(s_alloc(s.get(), &s->in[i].cert, HW));
    FAV_TRY(s_alloc(s.get(), &s->out[i], 3 * HW));
    FAV_TRY(check_cuda(cudaEventCreateWithFlags(&s->in[i].uploaded, cudaEventDisableTiming), "cudaEventCreate"));
    FAV_TRY(check_cuda(cudaEventCreateWithFlags(&s->in[i].consumed, cudaEventDisableTiming), "cudaEventCreate"));
    FAV_TRY(check_cuda(cudaEventCreateWithFlags(&s->computed[i], cudaEventDisableTiming), "cudaEventCreate"));
    FAV_TRY(check_cuda(cudaEventCreateWithFlags(&s->downloaded[i], cudaEventDisableTiming), "cudaEventCreate"));
  }
  for (int i = 0; i < fav_session::kDoneRing; ++i)  // waited on by host threads: block, do not spin
    FAV_TRY(check_cuda(cudaEventCreateWithFlags(&s->done[i], cudaEventDisableTiming | cudaEventBlockingSync), "cudaEventCreate"));
  FAV_TRY(check_cuda(cudaEventCreate(&s->t0), "cudaEventCreate"));
  FAV_TRY(check_cuda(cudaEventCreate(&s->t1), "cudaEventCreate"));
  *out = s.release();
  return FAV_OK;
}

// mode 0: first frame; 1: cert given; 2: cert from the flow pair; 3: cert from the flow pair and the frame (4-argument mode)
static int session_step(fav_session *s, int mode, const float *content_host, const float *flow_a, const float *flow_b,
                        const float *cert_host, int min_filter_r, int border_mode, float *out_host) {
  FAV_REQUIRE(s && content_host && out_host, "fav_session: null argument");
  FAV_REQUIRE(mode == 0 || s->have_prev, "fav_session_run_next_image: no previous frame (call run_image first)");
  FAV_REQUIRE(min_filter_r == 0 || ((min_filter_r & 1) && min_filter_r <= 15), "occlusions_min_filter must be odd <= 15");
  const int H = s->H, W = s->W;
  const size_t HW = (size_t)H * W;
  const int si = (int)(s->frame & 1), so = (int)(s->frame & 1);
  fav_session::InSet &in = s->in[si];
  // ---- H2D (waits until the frame that last used this input set has consumed it)
  if (in.used) FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_h2d, in.consumed, 0), "cudaStreamWaitEvent"));
  FAV_TRY(check_cuda(cudaMemcpyAsync(in.content, content_host, 3 * HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D content"));
  if (mode == 1) {
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.flow, flow_a, 2 * HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flow"));
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.cert_raw, cert_host, HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D cert"));
  } else if (mode >= 2) {
    // backward flow arrives in .flo order (u,v); the warp wants (dy,dx) = (v,u): swap planes while uploading
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.flow + HW, flow_a, HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flow u"));
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.flow, flow_a + HW, HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flow v"));
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.flow_fw, flow_b, 2 * HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flow fw"));
  }
  FAV_TRY(check_cuda(cudaEventRecord(in.uploaded, s->s_h2d), "cudaEventRecord"));
  // ---- compute
  FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_comp, in.uploaded, 0), "cudaStreamWaitEvent"));
  if (s->out_used[so])  // the D2H of the frame that last wrote out[so] must be finished
    FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_comp, s->downloaded[so], 0), "cudaStreamWaitEvent"));
  FAV_TRY(check_cuda(cudaEventRecord(s->t0, s->s_comp), "cudaEventRecord"));
  if (mode == 0) {
    FAV_TRY(fav_run_image(s->net_img ? s->net_img : s->net, in.content, nullptr, H, W, s->out[so], s->s_comp));
  } else if (mode == 3) {
    FAV_TRY(fav_run_next_image_flows_structure(s->net, in.content, s->out[so ^ 1], in.flow, in.flow_fw, nullptr, nullptr, H, W,
                                               min_filter_r, border_mode, s->out[so], s->s_comp));
  } else {
    // ONE temporal-stage kernel per frame: occlusion test (mode 2) or given certainty (mode 1) -> min filter -> warp ->
    // preprocess -> mask -> concat -> first operand of the net; then one graph launch
    FAV_TRY(fav_run_next_image_flows(s->net, in.content, s->out[so ^ 1], in.flow, mode == 2 ? in.flow_fw : nullptr,
                                     mode == 1 ? in.cert_raw : nullptr, nullptr, nullptr, H, W, min_filter_r, border_mode,
                                     s->out[so], s->s_comp));
  }
  FAV_TRY(check_cuda(cudaEventRecord(s->t1, s->s_comp), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(in.consumed, s->s_comp), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(s->computed[so], s->s_comp), "cudaEventRecord"));
  in.used = true;
  // ---- D2H
  FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_d2h, s->computed[so], 0), "cudaStreamWaitEvent"));
  FAV_TRY(check_cuda(cudaMemcpyAsync(out_host, s->out[so], 3 * HW * 4, cudaMemcpyDeviceToHost, s->s_d2h), "D2H out"));
  FAV_TRY(check_cuda(cudaEventRecord(s->downloaded[so], s->s_d2h), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(s->done[s->frame % fav_session::kDoneRing], s->s_d2h), "cudaEventRecord"));
  s->out_used[so] = true;
  s->have_prev = true;
  s->frame++;
  return FAV_OK;
}

int fav_session_set_image_model(fav_session_t *s, fav_net_t *net_img) {
  FAV_REQUIRE(s, "fav_session_set_image_model: null session");
  s->net_img = net_img;
  return FAV_OK;
}

int fav_session_run_image(fav_session_t *s, const float *content_host, float *out_host) {
  return session_step(s, 0, content_host, nullptr, nullptr, nullptr, 0, 0, out_host);
}

int fav_session_run_next_image(fav_session_t *s, const float *content_host, const float *flow_host,
                               const float *cert_host, int min_filter_r, int border_mode, float *out_host) {
  FAV_REQUIRE(flow_host && cert_host, "fav_session_run_next_image: null flow / cert");
  return session_step(s, 1, content_host, flow_host, nullptr, cert_host, min_filter_r, border_mode, out_host);
}

int fav_session_run_next_image_flows(fav_session_t *s, const float *content_host, const float *flow_bw_uv_host,
                                     const float *flow_fw_uv_host, int min_filter_r, int border_mode, float *out_host) {
  FAV_REQUIRE(flow_bw_uv_host && flow_fw_uv_host, "fav_session_run_next_image_flows: null flow");
  return session_step(s, 2, content_host, flow_bw_uv_host, flow_fw_uv_host, nullptr, min_filter_r, border_mode, out_host);
}

int fav_session_run_next_image_flows_structure(fav_session_t *s, const float *content_host, const float *flow_bw_uv_host,
                                               const float *flow_fw_uv_host, int min_filter_r, int border_mode, float *out_host) {
  FAV_REQUIRE(flow_bw_uv_host && flow_fw_uv_host, "fav_session_run_next_image_flows_structure: null flow");
  return session_step(s, 3, content_host, flow_bw_uv_host, flow_fw_uv_host, nullptr, min_filter_r, border_mode, out_host);
}

// The two conversions as device-pointer entry points (multi-GPU data plane: frames travel as the 8-bit pixels the files hold and
// are converted on the GPU that owns the clip).  Any of flo_uv / cert8 (and their outputs) may be NULL.
int fav_bytes_to_planes(const unsigned char *rgb_hwc, const float *flo_uv, const unsigned char *cert8, int invert_occlusion,
                        float *content, float *flow, float *cert, int H, int W, void *stream) {
  FAV_REQUIRE(rgb_hwc && content && H > 0 && W > 0, "fav_bytes_to_planes: bad argument");
  FAV_REQUIRE((flo_uv == nullptr) == (flow == nullptr) && (cert8 == nullptr) == (cert == nullptr), "fav_bytes_to_planes: input / output mismatch");
  FAV_TRY(require_device());
  const int64_t HW = (int64_t)H * W;
  decode_bytes_kernel<<<(unsigned)((HW + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rgb_hwc, (const float2 *)flo_uv, cert8, invert_occlusion,
                                                                                  content, flow, cert, HW, nullptr, nullptr);
  return post_launch("decode_bytes");
}

int fav_planes_to_png_rows(const float *rgb_planes, unsigned char *rows, int H, int W, void *stream) {
  FAV_REQUIRE(rgb_planes && rows && H > 0 && W > 0, "fav_planes_to_png_rows: bad argument");
  FAV_TRY(require_device());
  encode_rows_kernel<<<dim3((unsigned)((W + 255) / 256), (unsigned)H), 256, 0, (cudaStream_t)stream>>>(rgb_planes, rows, H, W);
  return post_launch("encode_rows");
}

// One frame from FILE PAYLOADS: rgb_hwc = the P6 payload (H*W*3 bytes), flo_uv = the .flo payload (H*W (u,v) float pairs) and
// cert8 = the P5 payload of the certainty (both NULL for the first frame / a single image); png_rows_host receives
// H*(1+3W) bytes of Sub-filtered PNG scanlines of the stylized frame.  The byte <-> float conversions run on the copy
// streams (decode after the H2D, encode before the D2H), the compute stream runs exactly what fav_session_run_next_image runs.
// flo_fw_uv != NULL (cert8 then NULL): the certainty in 4-argument mode from the two flows and the frame
// (fav_session_run_frame_bytes_flows)
static int frame_bytes_step(fav_session_t *s, const unsigned char *rgb_hwc, const float *flo_uv, const float *flo_fw_uv,
                            const unsigned char *cert8, int invert_occlusion, int min_filter_r, int border_mode,
                            unsigned char *png_rows_host) {
  const bool first = flo_uv == nullptr;
  FAV_REQUIRE(first || s->have_prev, "fav_session_run_frame_bytes: no previous frame");
  FAV_REQUIRE(min_filter_r == 0 || ((min_filter_r & 1) && min_filter_r <= 15), "occlusions_min_filter must be odd <= 15");
  const int H = s->H, W = s->W;
  const size_t HW = (size_t)H * W, row_bytes = (size_t)H * (1 + 3 * (size_t)W);
  const int si = (int)(s->frame & 1), so = si;
  fav_session::InSet &in = s->in[si];
  if (!in.rgb8) {
    for (int i = 0; i < 2; ++i) {
      void *d = nullptr;
      FAV_TRY(check_cuda(cudaMalloc(&d, 3 * HW), "cudaMalloc(session bytes)")); s->allocs.push_back(d); s->in[i].rgb8 = (unsigned char *)d;
      FAV_TRY(check_cuda(cudaMalloc(&d, HW), "cudaMalloc(session bytes)")); s->allocs.push_back(d); s->in[i].cert8 = (unsigned char *)d;
      FAV_TRY(check_cuda(cudaMalloc(&d, row_bytes), "cudaMalloc(session bytes)")); s->allocs.push_back(d); s->rows8[i] = (unsigned char *)d;
      FAV_TRY(s_alloc(s, &s->in[i].flo_uv, 2 * HW));
    }
  }
  if (flo_fw_uv && !in.flo_fw_uv)
    for (int i = 0; i < 2; ++i) FAV_TRY(s_alloc(s, &s->in[i].flo_fw_uv, 2 * HW));
  // ---- H2D + decode
  if (in.used) FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_h2d, in.consumed, 0), "cudaStreamWaitEvent"));
  FAV_TRY(check_cuda(cudaMemcpyAsync(in.rgb8, rgb_hwc, 3 * HW, cudaMemcpyHostToDevice, s->s_h2d), "H2D rgb"));
  if (!first) {
    FAV_TRY(check_cuda(cudaMemcpyAsync(in.flo_uv, flo_uv, 2 * HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flo"));
    if (cert8) FAV_TRY(check_cuda(cudaMemcpyAsync(in.cert8, cert8, HW, cudaMemcpyHostToDevice, s->s_h2d), "H2D cert"));
    if (flo_fw_uv)
      FAV_TRY(check_cuda(cudaMemcpyAsync(in.flo_fw_uv, flo_fw_uv, 2 * HW * 4, cudaMemcpyHostToDevice, s->s_h2d), "H2D flo fw"));
  }
  decode_bytes_kernel<<<(unsigned)((HW + 255) / 256), 256, 0, s->s_h2d>>>(in.rgb8, first ? nullptr : (const float2 *)in.flo_uv,
                                                                        cert8 ? in.cert8 : nullptr, invert_occlusion, in.content,
                                                                        in.flow, in.cert_raw, (int64_t)HW,
                                                                        flo_fw_uv ? (const float2 *)in.flo_fw_uv : nullptr,
                                                                        in.flow_fw);
  FAV_TRY(post_launch("decode_bytes"));
  FAV_TRY(check_cuda(cudaEventRecord(in.uploaded, s->s_h2d), "cudaEventRecord"));
  // ---- compute
  FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_comp, in.uploaded, 0), "cudaStreamWaitEvent"));
  if (s->out_used[so]) FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_comp, s->downloaded[so], 0), "cudaStreamWaitEvent"));
  FAV_TRY(check_cuda(cudaEventRecord(s->t0, s->s_comp), "cudaEventRecord"));
  if (first) {
    FAV_TRY(fav_run_image(s->net_img ? s->net_img : s->net, in.content, nullptr, H, W, s->out[so], s->s_comp));
  } else if (flo_fw_uv) {
    FAV_TRY(fav_run_next_image_flows_structure(s->net, in.content, s->out[so ^ 1], in.flow, in.flow_fw, nullptr, nullptr, H, W,
                                               min_filter_r, border_mode, s->out[so], s->s_comp));
  } else {
    FAV_TRY(fav_run_next_image_flows(s->net, in.content, s->out[so ^ 1], in.flow, nullptr, in.cert_raw, nullptr, nullptr, H, W,
                                     min_filter_r, border_mode, s->out[so], s->s_comp));
  }
  FAV_TRY(check_cuda(cudaEventRecord(s->t1, s->s_comp), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(in.consumed, s->s_comp), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(s->computed[so], s->s_comp), "cudaEventRecord"));
  in.used = true;
  // ---- encode + D2H (out[so] is read by the next frame's warp as well: reads only, no ordering needed between them)
  FAV_TRY(check_cuda(cudaStreamWaitEvent(s->s_d2h, s->computed[so], 0), "cudaStreamWaitEvent"));
  encode_rows_kernel<<<dim3((unsigned)((W + 255) / 256), (unsigned)H), 256, 0, s->s_d2h>>>(s->out[so], s->rows8[so], H, W);
  FAV_TRY(post_launch("encode_rows"));
  FAV_TRY(check_cuda(cudaMemcpyAsync(png_rows_host, s->rows8[so], row_bytes, cudaMemcpyDeviceToHost, s->s_d2h), "D2H rows"));
  FAV_TRY(check_cuda(cudaEventRecord(s->downloaded[so], s->s_d2h), "cudaEventRecord"));
  FAV_TRY(check_cuda(cudaEventRecord(s->done[s->frame % fav_session::kDoneRing], s->s_d2h), "cudaEventRecord"));
  s->out_used[so] = true;
  s->have_prev = true;
  s->frame++;
  return FAV_OK;
}

int fav_session_run_frame_bytes(fav_session_t *s, const unsigned char *rgb_hwc, const float *flo_uv, const unsigned char *cert8,
                                int invert_occlusion, int min_filter_r, int border_mode, unsigned char *png_rows_host) {
  FAV_REQUIRE(s && rgb_hwc && png_rows_host, "fav_session_run_frame_bytes: null argument");
  FAV_REQUIRE((flo_uv != nullptr) == (cert8 != nullptr), "fav_session_run_frame_bytes: flow and certainty come together");
  return frame_bytes_step(s, rgb_hwc, flo_uv, nullptr, cert8, invert_occlusion, min_filter_r, border_mode, png_rows_host);
}

int fav_session_run_frame_bytes_flows(fav_session_t *s, const unsigned char *rgb_hwc, const float *flo_bw_uv,
                                      const float *flo_fw_uv, int min_filter_r, int border_mode, unsigned char *png_rows_host) {
  FAV_REQUIRE(s && rgb_hwc && png_rows_host, "fav_session_run_frame_bytes_flows: null argument");
  FAV_REQUIRE((flo_bw_uv != nullptr) == (flo_fw_uv != nullptr), "fav_session_run_frame_bytes_flows: the two flows come together");
  return frame_bytes_step(s, rgb_hwc, flo_bw_uv, flo_fw_uv, nullptr, 0, min_filter_r, border_mode, png_rows_host);
}

// the stylized frame of call number `frame_index` (0-based count of run_* calls on this session) has landed in its out_host
// buffer; wait != 0 blocks until then.  One completion event per frame in a ring of 64: frames older than that have landed
// long ago (the ring slot then belongs to a later frame, and waiting for it is never too short).
int fav_session_frame_done(fav_session_t *s, uint64_t frame_index, int wait) {
  FAV_REQUIRE(s && frame_index < s->frame, "fav_session_frame_done: frame %llu was never enqueued", (unsigned long long)frame_index);
  cudaEvent_t ev = s->done[frame_index % fav_session::kDoneRing];
  if (wait) return check_cuda(cudaEventSynchronize(ev), "cudaEventSynchronize(frame done)");
  cudaError_t e = cudaEventQuery(ev);
  if (e == cudaSuccess) return FAV_OK;
  if (e == cudaErrorNotReady) { set_error("frame %llu still in flight", (unsigned long long)frame_index); return FAV_ERR_INVALID; }
  return check_cuda(e, "cudaEventQuery(frame done)");
}

int fav_session_sync(fav_session_t *s) {
  FAV_REQUIRE(s, "fav_session_sync: null session");
  FAV_TRY(check_cuda(cudaStreamSynchronize(s->s_h2d), "sync h2d"));
  FAV_TRY(check_cuda(cudaStreamSynchronize(s->s_comp), "sync compute"));
  return check_cuda(cudaStreamSynchronize(s->s_d2h), "sync d2h");
}

float fav_session_last_gpu_ms(fav_session_t *s) {
  if (!s || !s->t0 || !s->t1) return -1.f;
  if (cudaEventSynchronize(s->t1) != cudaSuccess) return -1.f;
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, s->t0, s->t1) != cudaSuccess) return -1.f;
  return ms;
}
}
