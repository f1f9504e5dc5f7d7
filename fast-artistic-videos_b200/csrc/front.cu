// front.cu -- the temporal-consistency front end (all HBM-bound, fp32, bit-exact vs oracle/fav_oracle.c):
//   a-1  nn.BilinearSamplerBDHW forward           stnbdhw/BilinearSamplerBDHW.cu:48-152
//   a-2  utils.warp_image                         fast_artistic_video/utils.lua:141-149
//   a-5  utils.min_filter                         fast_artistic_video/utils.lua:161-169
//   a-6  vgg preprocess / deprocess               fast_artistic_video/preprocess.lua:48-71
//   a-8  fused 7-channel temporal input           fast_artistic_video_core.lua:161-171
//   a-9  first-frame input                        fast_artistic_video_core.lua:133-137
//
// Design: one thread owns VEC (=4) consecutive output pixels of one row so that the flow,
// cert and content reads and all stores are 16-byte vector accesses, fully coalesced (the reference
// kernel maps lanes to x-stride-16 addresses and re-reads the flow once per channel).  The 4
// bilinear taps are scalar read-only loads; for real optical flow neighbouring lanes gather
// neighbouring addresses, so they coalesce in L1/L2 and each source sector is fetched from HBM once.
// All arithmetic uses explicit round-to-nearest intrinsics in the reference's evaluation order.  The bilinear
// blend reproduces the FMA contraction nvcc applies to the reference kernel (bilinear_ref_blend, fav_common.cuh), so the
// warp is bit-identical to the reference's own CUDA kernel compiled for sm_90a (oracle/ref_warp) and to the CPU oracle.
#include <algorithm>

#include "fav_common.cuh"
#include "net_layout.cuh"
#include "occlusion.cuh"

namespace fav {

// ---- shared per-pixel sampling ------------------------------------------------------------------
struct Sample {
  int x0, y0;
  float wx, wy;     // weights of the top-left corner (BilinearSamplerBDHW.cu:21-22)
  bool tl, tr, bl, br;
  bool off;         // PAD_PIXEL mode: whole pixel takes the pad value
  int x1, y1;       // PAD_PIXEL mode: clamped neighbours
};

__device__ __forceinline__ Sample make_sample(float dy, float dx, int yOut, int xOut, int H, int W,
                                              int border_mode) {
  Sample s;
  float yf = __fadd_rn(dy, (float)yOut);  // BilinearSamplerBDHW.cu:72
  float xf = __fadd_rn(dx, (float)xOut);  // :73
  float fy = floorf(yf), fx = floorf(xf);
  s.y0 = (int)fy;
  s.x0 = (int)fx;
  if (border_mode == FAV_BORDER_PER_TAP) {
    s.wx = __fsub_rn(1.0f, __fsub_rn(xf, (float)s.x0));  // :22
    s.wy = __fsub_rn(1.0f, __fsub_rn(yf, (float)s.y0));
    bool xin0 = s.x0 >= 0 && s.x0 <= W - 1, xin1 = s.x0 + 1 >= 0 && s.x0 + 1 <= W - 1;
    bool yin0 = s.y0 >= 0 && s.y0 <= H - 1, yin1 = s.y0 + 1 >= 0 && s.y0 + 1 <= H - 1;
    s.tl = xin0 && yin0;  // :92-95
    s.tr = xin1 && yin0;
    s.bl = xin0 && yin1;
    s.br = xin1 && yin1;
    s.off = false;
    s.x1 = s.x0 + 1;
    s.y1 = s.y0 + 1;
  } else {
    // image.warp(..., 'bilinear', true, 'pad', 0) (fast_artistic_video/utils.lua:147), see oracle
    s.off = (yf < 0.f || yf > (float)(H - 1) || xf < 0.f || xf > (float)(W - 1));
    s.wx = __fsub_rn(xf, (float)s.x0);  // here: fractional parts
    s.wy = __fsub_rn(yf, (float)s.y0);
    s.x1 = min(s.x0 + 1, W - 1);
    s.y1 = min(s.y0 + 1, H - 1);
    s.tl = s.tr = s.bl = s.br = !s.off;
  }
  return s;
}

__device__ __forceinline__ float sample_plane(const Sample &s, const float *__restrict__ p,
                                              int64_t sy, int64_t sx, int border_mode) {
  float vtl = 0.f, vtr = 0.f, vbl = 0.f, vbr = 0.f;
  if (s.tl) vtl = __ldg(p + (int64_t)s.y0 * sy + (int64_t)s.x0 * sx);
  if (s.tr) vtr = __ldg(p + (int64_t)s.y0 * sy + (int64_t)s.x1 * sx);
  if (s.bl) vbl = __ldg(p + (int64_t)s.y1 * sy + (int64_t)s.x0 * sx);
  if (s.br) vbr = __ldg(p + (int64_t)s.y1 * sy + (int64_t)s.x1 * sx);
  if (border_mode == FAV_BORDER_PER_TAP) {
    // BilinearSamplerBDHW.cu:103-106 with the FMA contraction of the compiled reference kernel (fav_common.cuh)
    float omx = __fsub_rn(1.0f, s.wx), omy = __fsub_rn(1.0f, s.wy);
    return bilinear_ref_blend(s.wx, s.wy, omx, omy, vtl, vtr, vbl, vbr);
  } else {
    if (s.off) return 0.0f;
    float omx = __fsub_rn(1.0f, s.wx), omy = __fsub_rn(1.0f, s.wy);
    float v = __fmul_rn(__fmul_rn(omy, omx), vtl);
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(omy, s.wx), vtr));
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(s.wy, omx), vbl));
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(s.wy, s.wx), vbr));
    return v;
  }
}

// same blend on taps already in registers (the fused kernels request every tap of a thread before using any)
__device__ __forceinline__ float blend_taps(const Sample &s, float vtl, float vtr, float vbl, float vbr, int border_mode) {
  const float omx = __fsub_rn(1.0f, s.wx), omy = __fsub_rn(1.0f, s.wy);
  if (border_mode == FAV_BORDER_PER_TAP) return bilinear_ref_blend(s.wx, s.wy, omx, omy, vtl, vtr, vbl, vbr);
  if (s.off) return 0.0f;
  float v = __fmul_rn(__fmul_rn(omy, omx), vtl);
  v = __fadd_rn(v, __fmul_rn(__fmul_rn(omy, s.wx), vtr));
  v = __fadd_rn(v, __fmul_rn(__fmul_rn(s.wy, omx), vbl));
  v = __fadd_rn(v, __fmul_rn(__fmul_rn(s.wy, s.wx), vbr));
  return v;
}

// ---- a-1: standalone warp ------------------------------------------------------------------------
struct Strides4 { int64_t b, c, h, w; };

// generic-stride kernel: one thread per output pixel, channels looped inside (flow read once)
__global__ void __launch_bounds__(256) warp_generic_kernel(
    const float *__restrict__ img, Strides4 is, const float *__restrict__ grid, Strides4 gs,
    float *__restrict__ out, Strides4 os, int C, int Hin, int Win, int Hout, int Wout, int border_mode) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  int b = blockIdx.z;
  if (x >= Wout || y >= Hout) return;
  const float *g = grid + b * gs.b + (int64_t)y * gs.h + (int64_t)x * gs.w;
  Sample s = make_sample(__ldg(g), __ldg(g + gs.c), y, x, Hin, Win, border_mode);
  for (int c = 0; c < C; ++c)
    out[b * os.b + c * os.c + (int64_t)y * os.h + (int64_t)x * os.w] =
        sample_plane(s, img + b * is.b + c * is.c, is.h, is.w, border_mode);
}

// contiguous-row fast path: 4 pixels / thread, float4 flow loads and float4 stores
template <int C_STATIC>
__global__ void __launch_bounds__(256) warp_vec4_kernel(
    const float *__restrict__ img, Strides4 is, const float *__restrict__ grid, Strides4 gs,
    float *__restrict__ out, Strides4 os, int C, int Hin, int Win, int Hout, int Wout, int border_mode) {
  int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  int b = blockIdx.z;
  if (x4 >= Wout || y >= Hout) return;
  const float *g = grid + b * gs.b + (int64_t)y * gs.h + x4;
  float4 dy = __ldg(reinterpret_cast<const float4 *>(g));
  float4 dx = __ldg(reinterpret_cast<const float4 *>(g + gs.c));
  Sample s0 = make_sample(dy.x, dx.x, y, x4 + 0, Hin, Win, border_mode);
  Sample s1 = make_sample(dy.y, dx.y, y, x4 + 1, Hin, Win, border_mode);
  Sample s2 = make_sample(dy.z, dx.z, y, x4 + 2, Hin, Win, border_mode);
  Sample s3 = make_sample(dy.w, dx.w, y, x4 + 3, Hin, Win, border_mode);
  const int Cn = C_STATIC > 0 ? C_STATIC : C;
#pragma unroll
  for (int c = 0; c < Cn; ++c) {
    const float *p = img + b * is.b + c * is.c;
    float4 v;
    v.x = sample_plane(s0, p, is.h, 1, border_mode);
    v.y = sample_plane(s1, p, is.h, 1, border_mode);
    v.z = sample_plane(s2, p, is.h, 1, border_mode);
    v.w = sample_plane(s3, p, is.h, 1, border_mode);
    __stcs(reinterpret_cast<float4 *>(out + b * os.b + c * os.c + (int64_t)y * os.h + x4), v);
  }
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int launch_warp(const float *img, const int64_t isz[4], const int64_t ist[4], const float *grid,
                       const int64_t gsz[4], const int64_t gst[4], float *out, const int64_t ost[4],
                       int border_mode, cudaStream_t st) {
  // the Lua asserts of BilinearSamplerBDHW:check (BilinearSamplerBDHW.lua:26-42)
  FAV_REQUIRE(img && grid && out, "BilinearSamplerBDHW: null tensor");
  FAV_REQUIRE(isz[0] == gsz[0], "BilinearSamplerBDHW: batch mismatch (%lld vs %lld)", (long long)isz[0],
              (long long)gsz[0]);
  FAV_REQUIRE(gsz[1] == 2, "BilinearSamplerBDHW: grids:size(2) must be 2 (got %lld)", (long long)gsz[1]);
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  for (int i = 0; i < 4; ++i) FAV_REQUIRE(isz[i] > 0 && gsz[i] > 0, "BilinearSamplerBDHW: empty tensor");
  FAV_TRY(require_device());
  int B = (int)isz[0], C = (int)isz[1], Hin = (int)isz[2], Win = (int)isz[3];
  int Hout = (int)gsz[2], Wout = (int)gsz[3];
  Strides4 is{ist[0], ist[1], ist[2], ist[3]}, gs{gst[0], gst[1], gst[2], gst[3]},
      os{ost[0], ost[1], ost[2], ost[3]};
  bool vec = is.w == 1 && gs.w == 1 && os.w == 1 && (Wout % 4 == 0) && aligned16(grid) && aligned16(out) &&
             (gs.b % 4 == 0) && (gs.c % 4 == 0) && (gs.h % 4 == 0) && (os.b % 4 == 0) && (os.c % 4 == 0) &&
             (os.h % 4 == 0);
  if (vec) {
    dim3 block(32, 8), gridDim(ceil_div(Wout / 4, 32), ceil_div(Hout, 8), B);
    if (C == 3)
      warp_vec4_kernel<3><<<gridDim, block, 0, st>>>(img, is, grid, gs, out, os, C, Hin, Win, Hout, Wout, border_mode);
    else if (C == 1)
      warp_vec4_kernel<1><<<gridDim, block, 0, st>>>(img, is, grid, gs, out, os, C, Hin, Win, Hout, Wout, border_mode);
    else
      warp_vec4_kernel<0><<<gridDim, block, 0, st>>>(img, is, grid, gs, out, os, C, Hin, Win, Hout, Wout, border_mode);
  } else {
    dim3 block(32, 8), gridDim(ceil_div(Wout, 32), ceil_div(Hout, 8), B);
    warp_generic_kernel<<<gridDim, block, 0, st>>>(img, is, grid, gs, out, os, C, Hin, Win, Hout, Wout, border_mode);
  }
  return post_launch("BilinearSamplerBDHW.updateOutput");
}

// ---- a-8 / a-9: fused temporal input ---------------------------------------------------------------
// out7: [7,H,W] fp32.  VEC pixels per thread.
// PACK: instead of the 7 fp32 planes, write the network's first operand directly (fp16 hi/lo, 8th channel zero) including
// the nn.SpatialReflectionPadding(R) copies (train_video.lua:319-324) -- what pack_input_kernel would produce from out7.
// Per-thread body: VEC consecutive pixels of row y starting at x0, certainty c[] already in registers (read from the cert
// plane by temporal_input_kernel, computed in shared memory by temporal_stage_kernel).
template <int VEC, bool FIRST, bool PACK>
__device__ __forceinline__ void temporal_pixels(
    const float *__restrict__ content, const float *__restrict__ prev, const float *__restrict__ flow,
    const float (&c)[VEC], const float *__restrict__ fill, const float *__restrict__ flow_mask,
    float *__restrict__ out7, int H, int W, int x0, int y, int border_mode, const Operand &dst, int R) {
  const int64_t HW = (int64_t)H * W;
  const int64_t o = (int64_t)y * W + x0;
  const float mean[3] = {FAV_MEAN_B, FAV_MEAN_G, FAV_MEAN_R};
  float cont[3][VEC], res[7][VEC];
  // content planes (R,G,B)
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    if (VEC == 4) {
      float4 t = __ldcs(reinterpret_cast<const float4 *>(content + j * HW + o));
      cont[j][0] = t.x; cont[j][1] = t.y; cont[j][2] = t.z; cont[j][3] = t.w;
    } else {
      cont[j][0] = __ldcs(content + j * HW + o);
    }
  }
  float dy[VEC], dx[VEC], fm[VEC];
  if (!FIRST) {
    if (VEC == 4) {
      float4 t = __ldg(reinterpret_cast<const float4 *>(flow + o));
      dy[0] = t.x; dy[1] = t.y; dy[2] = t.z; dy[3] = t.w;
      t = __ldg(reinterpret_cast<const float4 *>(flow + HW + o));
      dx[0] = t.x; dx[1] = t.y; dx[2] = t.z; dx[3] = t.w;
      if (flow_mask) {
        t = __ldcs(reinterpret_cast<const float4 *>(flow_mask + o));
        fm[0] = t.x; fm[1] = t.y; fm[2] = t.z; fm[3] = t.w;
      }
    } else {
      dy[0] = flow[o]; dx[0] = flow[HW + o];
      if (flow_mask) fm[0] = flow_mask[o];
    }
  }
  // all bilinear taps of the thread's pixels are requested before any of them is used (VEC x 3 planes x 4 corners
  // independent gathers in flight: the kernel is latency bound, not traffic bound)
  float wv[VEC][3];
  if (!FIRST) {
    Sample sm[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) sm[i] = make_sample(dy[i], dx[i], y, x0 + i, H, W, border_mode);
    float tap[VEC][3][4];
#pragma unroll
    for (int i = 0; i < VEC; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float *p = prev + k * HW;
        tap[i][k][0] = sm[i].tl ? __ldg(p + (int64_t)sm[i].y0 * W + sm[i].x0) : 0.f;
        tap[i][k][1] = sm[i].tr ? __ldg(p + (int64_t)sm[i].y0 * W + sm[i].x1) : 0.f;
        tap[i][k][2] = sm[i].bl ? __ldg(p + (int64_t)sm[i].y1 * W + sm[i].x0) : 0.f;
        tap[i][k][3] = sm[i].br ? __ldg(p + (int64_t)sm[i].y1 * W + sm[i].x1) : 0.f;
      }
#pragma unroll
    for (int i = 0; i < VEC; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) wv[i][k] = blend_taps(sm[i], tap[i][k][0], tap[i][k][1], tap[i][k][2], tap[i][k][3], border_mode);
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    // in[k] = 255*content[2-k] - mean[k]   (preprocess.lua:61; core.lua:168)
#pragma unroll
    for (int k = 0; k < 3; ++k) res[k][i] = __fsub_rn(__fmul_rn(cont[2 - k][i], 255.0f), mean[k]);
    if (FIRST) {
#pragma unroll
      for (int k = 0; k < 3; ++k) res[3 + k][i] = 0.0f;
      res[6][i] = 0.0f;  // core.lua:135-136: everything "uncertain"
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float pre = __fsub_rn(__fmul_rn(wv[i][2 - k], 255.0f), mean[k]);  // core.lua:166
        res[3 + k][i] = __fmul_rn(pre, c[i]);                               // :167
      }
      res[6][i] = flow_mask ? fminf(c[i], fm[i]) : c[i];  // :169 cmin
    }
  }
  if (fill) {  // generate_fill, core.lua:108-117 ('uniform-random' supplies the tensor; 'vgg-mean' = NULL)
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int i = 0; i < VEC; ++i) res[3 + k][i] = __fadd_rn(__ldg(fill + k * HW + o + i), res[3 + k][i]);
  } else if (!FIRST) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int i = 0; i < VEC; ++i) res[3 + k][i] = __fadd_rn(0.0f, res[3 + k][i]);  // torch.add(zeros, x)
  }
  if (PACK) {
    // padded row / column indices fed by source index i: i itself, -i (1 <= i <= R) and 2(n-1)-i (n-1-R <= i <= n-2)
    int ry[3], nry = 0;
    ry[nry++] = y;
    if (y >= 1 && y <= R) ry[nry++] = -y;
    if (y <= H - 2 && y >= H - 1 - R) ry[nry++] = 2 * (H - 1) - y;
    uint4 *hi = reinterpret_cast<uint4 *>(dst.hi), *lo = reinterpret_cast<uint4 *>(dst.lo);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const int x = x0 + i;
      const float v[8] = {res[0][i], res[1][i], res[2][i], res[3][i], res[4][i], res[5][i], res[6][i], 0.f};
      uint4 h, l;
      split_store8(v, &h, &l);
      int cx[3], ncx = 0;
      cx[ncx++] = x;
      if (x >= 1 && x <= R) cx[ncx++] = -x;
      if (x <= W - 2 && x >= W - 1 - R) cx[ncx++] = 2 * (W - 1) - x;
      for (int a = 0; a < nry; ++a)
        for (int b = 0; b < ncx; ++b) {
          const int64_t q = dst.off16(dst.padT + R + ry[a], 0, dst.padL + R + cx[b]);
          hi[q] = h; lo[q] = l;
        }
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    if (VEC == 4)
      *reinterpret_cast<float4 *>(out7 + k * HW + o) = make_float4(res[k][0], res[k][1], res[k][2], res[k][3]);
    else
      out7[k * HW + o] = res[k][0];
  }
}

// a batch of images (blockIdx.z = image b): every plane argument holds one image after the other, dst is image b of the operand
template <class T>
__device__ __forceinline__ T *img_plane(T *p, int b, int64_t per_image) { return p ? p + b * per_image : p; }

template <int VEC, bool FIRST, bool PACK = false>
__global__ void __launch_bounds__(256) temporal_input_kernel(
    const float *__restrict__ content, const float *__restrict__ prev, const float *__restrict__ flow,
    const float *__restrict__ cert, const float *__restrict__ fill, const float *__restrict__ flow_mask,
    float *__restrict__ out7, int H, int W, int border_mode, Operand dst = Operand(), int R = 0) {
  int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x0 >= W || y >= H) return;
  if (const int b = blockIdx.z) {
    const int64_t HW = (int64_t)H * W;
    content = img_plane(content, b, 3 * HW); prev = img_plane(prev, b, 3 * HW); flow = img_plane(flow, b, 2 * HW);
    cert = img_plane(cert, b, HW); fill = img_plane(fill, b, 3 * HW); flow_mask = img_plane(flow_mask, b, HW);
    out7 = img_plane(out7, b, 7 * HW);
    dst = image_of(dst, b);
  }
  const int64_t o = (int64_t)y * W + x0;
  float c[VEC];
  if (!FIRST) {
    if (VEC == 4) {
      const float4 t = __ldcs(reinterpret_cast<const float4 *>(cert + o));
      c[0] = t.x; c[1] = t.y; c[2] = t.z; c[3] = t.w;
    } else {
      c[0] = cert[o];
    }
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) c[i] = 0.f;
  }
  temporal_pixels<VEC, FIRST, PACK>(content, prev, flow, c, fill, flow_mask, out7, H, W, x0, y, border_mode, dst, R);
}

// ---- the WHOLE temporal-consistency stage in one kernel ---------------------------------------------------------------
// north star: "BilinearSamplerBDHW warp of the previous stylized frame by the supplied optical flow, consistencyChecker's
// forward/backward-flow occlusion test, and the channel concat ... become one fused sm_90a kernel ... that writes the
// 7-channel tensor the net consumes directly".  Per 64 x 16 pixel tile (256 threads x 4 pixels):
//   1. certainty of the tile + a (r/2)-pixel halo into shared memory: MODE 0 = the occlusion test itself
//      (consistencyChecker.cpp:99-125, 3-argument mode; flow1 = the backward flow that also drives the warp, flow2 = forward
//      flow) -- halo pixels are recomputed instead of exchanged; MODE 1 = a given certainty plane (func_load_cert output);
//      MODE 2 = MODE 0 in 4-argument mode (consistencyChecker.cpp:122-124, makeOptFlow_deepflow.sh:58-60): the structure term
//      from the corners plane and the device average of fav_compute_corners;
//   2. utils.min_filter (utils.lua:161-169) as a separable r x r minimum in shared memory (pad cells = +inf);
//   3. warp + preprocess + mask + concat of the thread's 4 pixels (temporal_pixels above).
// Bit-identical to consistency_kernel -> min_filter_kernel -> temporal_input_kernel (tests/test_gpu_front.py).
constexpr int TS_TX = 64, TS_TY = 16, TS_MAXP = 7;  // (64 x 32 tiles: 1.30x instead of 1.50x halo evaluations, but measured slower: 50.2 vs 47.5 us)
template <bool PACK, int MODE>
__global__ void __launch_bounds__(256) temporal_stage_kernel(
    const float *__restrict__ content, const float *__restrict__ prev, const float *__restrict__ flow,
    const float *__restrict__ fw_u, const float *__restrict__ fw_v, const float *__restrict__ cert_raw,
    const float *__restrict__ fill, const float *__restrict__ flow_mask, float *__restrict__ out7,
    float *__restrict__ cert_out, int H, int W, int r, int border_mode, Operand dst, int R,
    const float *__restrict__ structure, const float *__restrict__ structure_avg) {
  __shared__ float cs[TS_TY + 2 * TS_MAXP][TS_TX + 2 * TS_MAXP + 1];
  __shared__ float rm[TS_TY + 2 * TS_MAXP][TS_TX + 1];
  const int p = r / 2, bx = blockIdx.x * TS_TX, by = blockIdx.y * TS_TY;
  const int tw = TS_TX + 2 * p, th = TS_TY + 2 * p;
  const int64_t HW = (int64_t)H * W;
  if (const int b = blockIdx.z) {  // a batch: image b of every plane (img_plane) and of the operand
    content = img_plane(content, b, 3 * HW); prev = img_plane(prev, b, 3 * HW); flow = img_plane(flow, b, 2 * HW);
    fw_u = img_plane(fw_u, b, 2 * HW); fw_v = img_plane(fw_v, b, 2 * HW); cert_raw = img_plane(cert_raw, b, HW);
    fill = img_plane(fill, b, 3 * HW); flow_mask = img_plane(flow_mask, b, HW); out7 = img_plane(out7, b, 7 * HW);
    cert_out = img_plane(cert_out, b, HW);
    dst = image_of(dst, b);
  }
  if (MODE == 0 || MODE == 2) {
    const float savg = MODE == 2 ? __ldg(structure_avg) : 0.f;
    // kTsBatch pixels per thread and pass: first the (coalesced) backward-flow loads of all of them, then all their forward-flow
    // gathers, then the arithmetic -- up to 8 * kTsBatch loads in flight per thread instead of one pixel's dependent chain
    constexpr int kTsBatch = 3;
    for (int i0 = threadIdx.x; i0 < tw * th; i0 += 256 * kTsBatch) {
      int gx[kTsBatch], gy[kTsBatch], ty[kTsBatch], tx[kTsBatch];
      float u2[kTsBatch], v2[kTsBatch];
      bool in[kTsBatch];
#pragma unroll
      for (int k = 0; k < kTsBatch; ++k) {
        const int i = i0 + k * 256;
        ty[k] = i / tw; tx[k] = i - ty[k] * tw;
        gy[k] = by + ty[k] - p; gx[k] = bx + tx[k] - p;
        in[k] = i < tw * th && gy[k] >= 0 && gy[k] < H && gx[k] >= 0 && gx[k] < W;
        u2[k] = v2[k] = 0.f;
        if (in[k]) {  // flow = (dy, dx) = (v, u) of the backward flow = flow1 of the checker
          const int64_t o = (int64_t)gy[k] * W + gx[k];
          u2[k] = __ldg(flow + HW + o); v2[k] = __ldg(flow + o);
        }
      }
      CheckTaps t[kTsBatch];
#pragma unroll
      for (int k = 0; k < kTsBatch; ++k) {
        t[k].inside = false;
        if (in[k]) t[k] = check_load(fw_u, fw_v, u2[k], v2[k], gx[k], gy[k], W, H);
      }
#pragma unroll
      for (int k = 0; k < kTsBatch; ++k) {
        if (i0 + k * 256 >= tw * th) break;
        // outside the image: ignored by the max-pooling of utils.min_filter (-inf padding)
        cs[ty[k]][tx[k]] = in[k] ? (check_eval(t[k], u2[k], v2[k], gx[k], gy[k], W, MODE == 2 ? structure : nullptr, savg) ? 1.f : 0.f) : INFINITY;
      }
    }
  } else {
    for (int i = threadIdx.x; i < tw * th; i += 256) {
      const int ty = i / tw, tx = i - ty * tw;
      const int gy = by + ty - p, gx = bx + tx - p;
      float v = INFINITY;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(cert_raw + (int64_t)gy * W + gx);
      cs[ty][tx] = v;
    }
  }
  __syncthreads();
  if (p > 0) {
    for (int i = threadIdx.x; i < th * TS_TX; i += 256) {
      const int ty = i / TS_TX, tx = i % TS_TX;
      float m = INFINITY;
      for (int d = 0; d < r; ++d) m = fminf(m, cs[ty][tx + d]);
      rm[ty][tx] = m;
    }
    __syncthreads();
  }
  const int tx4 = (threadIdx.x & 15) * 4, x0 = bx + tx4;
  if (x0 >= W) return;
#pragma unroll 1
  for (int ty = threadIdx.x >> 4; ty < TS_TY; ty += 16) {
    const int y = by + ty;
    if (y >= H) return;
    float c[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (p > 0) {
        float m = INFINITY;
        for (int d = 0; d < r; ++d) m = fminf(m, rm[ty + d][tx4 + i]);
        // MulConstant(-1), AddConstant(1), pool, MulConstant(-1), AddConstant(1)  (utils.lua:162-167)
        const float t = __fadd_rn(__fmul_rn(m, -1.0f), 1.0f);
        c[i] = __fadd_rn(__fmul_rn(t, -1.0f), 1.0f);
      } else {
        c[i] = cs[ty][tx4 + i];
      }
    }
    if (cert_out) *reinterpret_cast<float4 *>(cert_out + (int64_t)y * W + x0) = make_float4(c[0], c[1], c[2], c[3]);
    temporal_pixels<4, false, PACK>(content, prev, flow, c, fill, flow_mask, out7, H, W, x0, y, border_mode, dst, R);
  }
}

// run_[next_]image: the fused input written straight into the first operand of the network (no out7 round trip)
int launch_temporal_input_packed(const float *content, const float *prev, const float *flow, const float *cert,
                                 const float *fill, const float *flow_mask, const Operand &dst, int R, int H, int W,
                                 int border_mode, bool first, cudaStream_t st, int nimg = 1) {
  const bool vec = (W % 4 == 0) && aligned16(content) && (first || (aligned16(flow) && aligned16(cert))) &&
                   (!flow_mask || aligned16(flow_mask)) && (!fill || aligned16(fill));
  dim3 block(32, 8);
  if (vec) {
    dim3 grid(ceil_div(W / 4, 32), ceil_div(H, 8), nimg);
    if (first)
      temporal_input_kernel<4, true, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, nullptr, H, W, border_mode, dst, R);
    else
      temporal_input_kernel<4, false, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, nullptr, H, W, border_mode, dst, R);
  } else {
    dim3 grid(ceil_div(W, 32), ceil_div(H, 8), nimg);
    if (first)
      temporal_input_kernel<1, true, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, nullptr, H, W, border_mode, dst, R);
    else
      temporal_input_kernel<1, false, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, nullptr, H, W, border_mode, dst, R);
  }
  return post_launch(first ? "first_frame_input" : "temporal_input");
}

// the whole stage in one launch.  Exactly one of (fw_uv, cert_raw) is non-null.  dst != null: write the network's first
// operand (PACK), else the 7 fp32 planes out7.  Returns FAV_ERR_UNSUPPORTED when the 16-byte vector path does not apply
// (callers then fall back to the three separate kernels).
int launch_temporal_stage(const float *content, const float *prev, const float *flow, const float *fw_uv, const float *cert_raw,
                          const float *fill, const float *flow_mask, float *out7, float *cert_out, const Operand *dst, int R,
                          int H, int W, int r, int border_mode, cudaStream_t st, int nimg = 1) {
  const bool vec = (W % 4 == 0) && aligned16(content) && aligned16(flow) && (!flow_mask || aligned16(flow_mask)) &&
                   (!fill || aligned16(fill)) && (!out7 || aligned16(out7)) && (!cert_out || aligned16(cert_out));
  if (!vec || r < 0 || r / 2 > TS_MAXP || (r > 1 && !(r & 1))) return FAV_ERR_UNSUPPORTED;
  const int64_t HW = (int64_t)H * W;
  dim3 grid(ceil_div(W, TS_TX), ceil_div(H, TS_TY), nimg);
  const Operand d = dst ? *dst : Operand();
  if (fw_uv) {
    if (dst) temporal_stage_kernel<true, 0><<<grid, 256, 0, st>>>(content, prev, flow, fw_uv, fw_uv + HW, nullptr, fill, flow_mask, nullptr, cert_out, H, W, r, border_mode, d, R, nullptr, nullptr);
    else temporal_stage_kernel<false, 0><<<grid, 256, 0, st>>>(content, prev, flow, fw_uv, fw_uv + HW, nullptr, fill, flow_mask, out7, cert_out, H, W, r, border_mode, d, R, nullptr, nullptr);
  } else {
    if (dst) temporal_stage_kernel<true, 1><<<grid, 256, 0, st>>>(content, prev, flow, nullptr, nullptr, cert_raw, fill, flow_mask, nullptr, cert_out, H, W, r, border_mode, d, R, nullptr, nullptr);
    else temporal_stage_kernel<false, 1><<<grid, 256, 0, st>>>(content, prev, flow, nullptr, nullptr, cert_raw, fill, flow_mask, out7, cert_out, H, W, r, border_mode, d, R, nullptr, nullptr);
  }
  return post_launch("temporal_stage");
}

// the stage in 4-argument mode (MODE 2), writing the network's first operand; one image
int launch_temporal_stage_structure(const float *content, const float *prev, const float *flow, const float *fw_uv,
                                    const float *structure, const float *structure_avg, const float *fill, const float *flow_mask,
                                    float *cert_out, const Operand &dst, int R, int H, int W, int r, int border_mode, cudaStream_t st) {
  const bool vec = (W % 4 == 0) && aligned16(content) && aligned16(flow) && (!flow_mask || aligned16(flow_mask)) &&
                   (!fill || aligned16(fill)) && (!cert_out || aligned16(cert_out));
  if (!vec || r < 0 || r / 2 > TS_MAXP || (r > 1 && !(r & 1))) return FAV_ERR_UNSUPPORTED;
  const int64_t HW = (int64_t)H * W;
  dim3 grid(ceil_div(W, TS_TX), ceil_div(H, TS_TY), 1);
  temporal_stage_kernel<true, 2><<<grid, 256, 0, st>>>(content, prev, flow, fw_uv, fw_uv + HW, nullptr, fill, flow_mask, nullptr,
                                                       cert_out, H, W, r, border_mode, dst, R, structure, structure_avg);
  return post_launch("temporal_stage.structure");
}

int launch_temporal_input(const float *content, const float *prev, const float *flow, const float *cert,
                          const float *fill, const float *flow_mask, float *out7, int H, int W,
                          int border_mode, bool first, cudaStream_t st, int nimg = 1) {
  bool vec = (W % 4 == 0) && aligned16(content) && aligned16(out7) && (first || (aligned16(flow) && aligned16(cert))) &&
             (!flow_mask || aligned16(flow_mask));
  dim3 block(32, 8);
  if (vec) {
    dim3 grid(ceil_div(W / 4, 32), ceil_div(H, 8), nimg);
    if (first)
      temporal_input_kernel<4, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, out7, H, W, border_mode);
    else
      temporal_input_kernel<4, false><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, out7, H, W, border_mode);
  } else {
    dim3 grid(ceil_div(W, 32), ceil_div(H, 8), nimg);
    if (first)
      temporal_input_kernel<1, true><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, out7, H, W, border_mode);
    else
      temporal_input_kernel<1, false><<<grid, block, 0, st>>>(content, prev, flow, cert, fill, flow_mask, out7, H, W, border_mode);
  }
  return post_launch(first ? "first_frame_input" : "temporal_input");
}

// ---- a-5: min filter -------------------------------------------------------------------------------
// 1 - maxpool_{r x r,s1,p=r/2}(1 - x) == fl(1 - fl(1 - min_window(x))) (rounding is monotone); pad cells
// are ignored by max-pooling (-inf padding), i.e. +inf for the min.
#define MF_TX 64
#define MF_TY 16
#define MF_MAXP 7
__global__ void __launch_bounds__(256) min_filter_kernel(const float *__restrict__ in, float *__restrict__ out,
                                                         int H, int W, int r) {
  __shared__ float tile[MF_TY + 2 * MF_MAXP][MF_TX + 2 * MF_MAXP + 1];
  __shared__ float rowmin[MF_TY + 2 * MF_MAXP][MF_TX + 1];
  const int p = r / 2;
  const int bx = blockIdx.x * MF_TX, by = blockIdx.y * MF_TY;
  const float *src = in + (int64_t)blockIdx.z * H * W;
  float *dst = out + (int64_t)blockIdx.z * H * W;
  const int tw = MF_TX + 2 * p, th = MF_TY + 2 * p;
  for (int i = threadIdx.x; i < tw * th; i += blockDim.x) {
    int ty = i / tw, tx = i % tw;
    int gy = by + ty - p, gx = bx + tx - p;
    tile[ty][tx] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(src + (int64_t)gy * W + gx) : INFINITY;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < th * MF_TX; i += blockDim.x) {
    int ty = i / MF_TX, tx = i % MF_TX;
    float m = INFINITY;
    for (int d = 0; d < r; ++d) m = fminf(m, tile[ty][tx + d]);
    rowmin[ty][tx] = m;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < MF_TY * MF_TX; i += blockDim.x) {
    int ty = i / MF_TX, tx = i % MF_TX;
    int gy = by + ty, gx = bx + tx;
    if (gy >= H || gx >= W) continue;
    float m = INFINITY;
    for (int d = 0; d < r; ++d) m = fminf(m, rowmin[ty + d][tx]);
    // MulConstant(-1), AddConstant(1), pool, MulConstant(-1), AddConstant(1)  (utils.lua:162-167)
    float t = __fadd_rn(__fmul_rn(m, -1.0f), 1.0f);
    dst[(int64_t)gy * W + gx] = __fadd_rn(__fmul_rn(t, -1.0f), 1.0f);
  }
}

int launch_min_filter(const float *in, float *out, int n, int H, int W, int r, cudaStream_t st) {
  dim3 grid(ceil_div(W, MF_TX), ceil_div(H, MF_TY), n);
  min_filter_kernel<<<grid, 256, 0, st>>>(in, out, H, W, r);
  return post_launch("min_filter");
}

// ---- a-6: vgg pre/deprocess ------------------------------------------------------------------------
template <bool DE>
__global__ void __launch_bounds__(256) vgg_kernel(const float *__restrict__ in, float *__restrict__ out, int64_t HW,
                                                  int64_t total_px) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total_px) return;
  int64_t n = i / HW, px = i % HW;
  const float *src = in + n * 3 * HW + px;
  float *dst = out + n * 3 * HW + px;
  const float mean[3] = {FAV_MEAN_B, FAV_MEAN_G, FAV_MEAN_R};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (!DE)
      dst[k * HW] = __fsub_rn(__fmul_rn(src[(2 - k) * HW], 255.0f), mean[k]);  // preprocess.lua:61
    else
      dst[(2 - k) * HW] = __fdiv_rn(__fadd_rn(src[k * HW], mean[k]), 255.0f);  // :70
  }
}

// ---- f-4: temporal loss of -evaluate (fast_artistic_video.lua:128-151) -------------------------------------------------
// nn.MSECriterion(cmul(warp(prev_stylized, flow_eval), cert), cmul(stylized, cert)): one fused pass (warp + mask + squared
// difference + reduction) instead of a warp, two cmuls and the criterion; the sum of squares is accumulated in double.
__global__ void __launch_bounds__(256) temporal_mse_kernel(const float *__restrict__ prev, const float *__restrict__ cur,
                                                           const float *__restrict__ flow, const float *__restrict__ cert,
                                                           int H, int W, int border_mode, double *__restrict__ sum) {
  const int64_t HW = (int64_t)H * W;
  double acc = 0.0;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < HW; o += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(o / W), x = (int)(o - (int64_t)y * W);
    const Sample s = make_sample(__ldg(flow + o), __ldg(flow + HW + o), y, x, H, W, border_mode);
    const float c = __ldg(cert + o);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float a = __fmul_rn(sample_plane(s, prev + k * HW, W, 1, border_mode), c), b = __fmul_rn(__ldg(cur + k * HW + o), c);
      const float d = __fsub_rn(a, b);
      acc += (double)d * (double)d;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  __shared__ double red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(sum, t);
  }
}

}  // namespace fav

using namespace fav;

extern "C" {

int fav_temporal_mse(const float *prev, const float *cur, const float *flow, const float *cert, int H, int W, int border_mode,
                     double *sum_dev, void *stream) {
  FAV_REQUIRE(prev && cur && flow && cert && sum_dev, "temporal_mse: null tensor");
  FAV_REQUIRE(H > 0 && W > 0, "temporal_mse: empty frame");
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  FAV_TRY(require_device());
  const int64_t HW = (int64_t)H * W;
  const int blocks = (int)std::min<int64_t>(ceil_div64(HW, 256), 148 * 8);
  temporal_mse_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(prev, cur, flow, cert, H, W, border_mode, sum_dev);
  return post_launch("temporal_mse");
}

int fav_bilinear_sampler_bdhw_update_output(const float *img, const int64_t img_size[4], const int64_t img_stride[4],
                                            const float *grid, const int64_t grid_size[4],
                                            const int64_t grid_stride[4], float *out, const int64_t out_stride[4],
                                            int border_mode, void *stream) {
  return launch_warp(img, img_size, img_stride, grid, grid_size, grid_stride, out, out_stride, border_mode,
                     (cudaStream_t)stream);
}

int fav_bilinear_sampler_bdhw_update_grad_input(void) {
  // BilinearSamplerBDHW.cu:171-176
  set_error("error in BilinearSampler.updateGradInput: Not implemented");
  return FAV_ERR_NOT_IMPLEMENTED;
}
int fav_bilinear_sampler_bdhw_update_grad_input_only_grid(void) {
  // BilinearSamplerBDHW.cu:179-184
  set_error("error in BilinearSampler.updateGradInput: Not implemented");
  return FAV_ERR_NOT_IMPLEMENTED;
}

int fav_warp_image(const float *img, int C, int Hin, int Win, const float *flow, int Hout, int Wout, float *out,
                   int border_mode, void *stream) {
  int64_t isz[4] = {1, C, Hin, Win}, ist[4] = {(int64_t)C * Hin * Win, (int64_t)Hin * Win, Win, 1};
  int64_t gsz[4] = {1, 2, Hout, Wout}, gst[4] = {(int64_t)2 * Hout * Wout, (int64_t)Hout * Wout, Wout, 1};
  int64_t ost[4] = {(int64_t)C * Hout * Wout, (int64_t)Hout * Wout, Wout, 1};
  return launch_warp(img, isz, ist, flow, gsz, gst, out, ost, border_mode, (cudaStream_t)stream);
}

int fav_min_filter(const float *in, float *out, int n, int H, int W, int r, void *stream) {
  FAV_REQUIRE(in && out, "min_filter: null tensor");
  FAV_REQUIRE(n > 0 && H > 0 && W > 0, "min_filter: empty tensor");
  FAV_REQUIRE(r >= 1 && (r & 1) && r / 2 <= MF_MAXP, "min_filter: r must be odd and <= %d", 2 * MF_MAXP + 1);
  FAV_TRY(require_device());
  return launch_min_filter(in, out, n, H, W, r, (cudaStream_t)stream);
}

int fav_vgg_preprocess(const float *in, float *out, int N, int H, int W, void *stream) {
  FAV_REQUIRE(in && out && N > 0 && H > 0 && W > 0, "vgg.preprocess: img must be N x 3 x H x W");
  FAV_TRY(require_device());
  int64_t HW = (int64_t)H * W, total = HW * N;
  vgg_kernel<false><<<(unsigned)ceil_div64(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, HW, total);
  return post_launch("vgg.preprocess");
}
int fav_vgg_deprocess(const float *in, float *out, int N, int H, int W, void *stream) {
  FAV_REQUIRE(in && out && N > 0 && H > 0 && W > 0, "vgg.deprocess: img must be N x 3 x H x W");
  FAV_TRY(require_device());
  int64_t HW = (int64_t)H * W, total = HW * N;
  vgg_kernel<true><<<(unsigned)ceil_div64(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, HW, total);
  return post_launch("vgg.deprocess");
}

int fav_temporal_input(const float *content, const float *prev, const float *flow, const float *cert,
                       const float *fill, const float *flow_mask, float *out7, int H, int W, int border_mode,
                       void *stream) {
  FAV_REQUIRE(content && prev && flow && cert && out7, "temporal_input: null tensor");
  FAV_REQUIRE(H > 0 && W > 0, "temporal_input: empty frame");
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  FAV_TRY(require_device());
  return launch_temporal_input(content, prev, flow, cert, fill, flow_mask, out7, H, W, border_mode, false,
                               (cudaStream_t)stream);
}

int fav_temporal_stage(const float *content, const float *prev, const float *flow_bw, const float *flow_fw_uv,
                       const float *cert_raw, const float *fill, const float *flow_mask, float *out7, float *cert_out,
                       int H, int W, int min_filter_r, int border_mode, void *stream) {
  FAV_REQUIRE(content && prev && flow_bw && out7, "temporal_stage: null tensor");
  FAV_REQUIRE((flow_fw_uv != nullptr) != (cert_raw != nullptr), "temporal_stage: give either the forward flow or a certainty plane");
  FAV_REQUIRE(H > 0 && W > 0, "temporal_stage: empty frame");
  FAV_REQUIRE(min_filter_r >= 0 && (min_filter_r <= 1 || (min_filter_r & 1)) && min_filter_r / 2 <= TS_MAXP,
              "temporal_stage: occlusions_min_filter must be odd and <= %d", 2 * TS_MAXP + 1);
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  FAV_TRY(require_device());
  int rc = launch_temporal_stage(content, prev, flow_bw, flow_fw_uv, cert_raw, fill, flow_mask, out7, cert_out, nullptr, 0, H, W,
                                 min_filter_r, border_mode, (cudaStream_t)stream);
  if (rc == FAV_ERR_UNSUPPORTED) set_error("temporal_stage: needs W %% 4 == 0 and 16-byte aligned planes");
  return rc;
}

int fav_first_frame_input(const float *content, const float *fill, float *out7, int H, int W, void *stream) {
  FAV_REQUIRE(content && out7, "first_frame_input: null tensor");
  FAV_REQUIRE(H > 0 && W > 0, "first_frame_input: empty frame");
  FAV_TRY(require_device());
  return launch_temporal_input(content, nullptr, nullptr, nullptr, fill, nullptr, out7, H, W, 0, true,
                               (cudaStream_t)stream);
}
}
