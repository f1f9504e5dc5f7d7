// percep.cu -- the perceptual loss network of -evaluate: content and style losses through a VGG-style loss network.
//   nn.PerceptualCriterion (setup, setStyleTarget, updateOutput)   fast_artistic_video/PerceptualCriterion.lua:27-155
//   nn.ContentLoss / nn.StyleLoss / nn.GramMatrix                  ContentLoss.lua:39-48, StyleLoss.lua:39-55, GramMatrix.lua:31-53
//   layer_utils.insert_after / trim_network                         layer_utils.lua:118-165
//   evaluate_image                                                  fast_artistic_video_core.lua:101-106
//
// The network is a chain of convolutions, ReLUs and max-poolings (the loss network trimmed after its deepest loss layer).
// Every convolution runs on conv_tc_kernel (wgmma implicit GEMM, fp16 hi/lo operands, three MMAs per K step); layers with
// more than 128 output channels run as one job per 128-channel N block (conv_plan.hpp).  After each convolution one
// kernel turns the raw fp32 output (bias included) into what follows: ReLU and max-pooling applied while the values are
// gathered, then the fp16 hi/lo split, written either as the next convolution's operand (zero border included) or as the
// feature map of a loss layer ("tap").
//
// A tap is stored pixel-contiguous per channel: [P/8 blocks][Cp channels][8 pixels] fp16 (hi and lo planes), Cp = C rounded
// up to 64, P = H*W padded with zeros to whole 128-pixel chunks.  For the Gram matrix F F^T, which contracts over pixels, this
// is the canonical no-swizzle K-major wgmma layout (8 channels x 8 pixels per 128-byte core matrix), the same descriptor form
// conv_tc_kernel uses for its operands, so one bulk copy per (8-pixel block, 64 channels) lands MMA-ready in shared memory.
//
// Values above the fp16 range (|x| > 65504) cannot be represented by the hi/lo pair (cvt.satfinite clamps them): the pack
// kernels count them, and an evaluation that met any returns an error instead of a loss computed from clamped features.
//
// Determinism: every sum has a fixed order -- Gram partial sums per (pixel range, tile) are added in split order in double,
// reductions use fixed grids and fixed shared-memory trees.
#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <vector>

#include "conv_plan.hpp"
#include "tc_common.cuh"
#include "wgmma_f16.cuh"

namespace fav {

// ---------------------------------------------------------------------------------------------------------------------
// device side
struct PoolSpec {
  int on, kw, kh, sw, sh, pw, ph;
};

// 8 channels (block cb) of pixel (y, x) of the stage output: max over the pooling window of the raw conv output, then ReLU.
// max-pooling and ReLU commute (ReLU is monotone; pooling pads with -inf), so one gather serves either module order.
__device__ __forceinline__ void gather8(const float4 *__restrict__ raw, int Cq, int Wp, int Hin, int Win, int y, int x, int cb,
                                        int relu, const PoolSpec &pl, float v[8]) {
  const bool q1 = 2 * cb + 1 < Cq;
  if (!pl.on) {
    const float4 a = __ldg(raw + ((int64_t)y * Cq + 2 * cb) * Wp + x);
    const float4 b = q1 ? __ldg(raw + ((int64_t)y * Cq + 2 * cb + 1) * Wp + x) : make_float4(0.f, 0.f, 0.f, 0.f);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = -INFINITY;
    const int hs = y * pl.sh - pl.ph, ws = x * pl.sw - pl.pw;
    const int he = min(hs + pl.kh, Hin), we = min(ws + pl.kw, Win);
    for (int iy = max(hs, 0); iy < he; ++iy)
      for (int ix = max(ws, 0); ix < we; ++ix) {
        const float4 a = __ldg(raw + ((int64_t)iy * Cq + 2 * cb) * Wp + ix);
        const float4 b = q1 ? __ldg(raw + ((int64_t)iy * Cq + 2 * cb + 1) * Wp + ix) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[0] = fmaxf(v[0], a.x); v[1] = fmaxf(v[1], a.y); v[2] = fmaxf(v[2], a.z); v[3] = fmaxf(v[3], a.w);
        v[4] = fmaxf(v[4], b.x); v[5] = fmaxf(v[5], b.y); v[6] = fmaxf(v[6], b.z); v[7] = fmaxf(v[7], b.w);
      }
  }
  if (relu)
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
}

__device__ __forceinline__ int out_of_fp16(float a) { return fabsf(a) > 65504.f ? 1 : 0; }  // also counts inf / NaN

__device__ __forceinline__ void flush_count(int cnt, int *counter) {
  if (cnt) atomicAdd(counter, cnt);
}

// VGG preprocess (preprocess.lua:57-62: RGB -> BGR, x255, - mean; the same fp32 operations as fav_vgg_preprocess) fused into
// the fp16 hi/lo pack of the first convolution's operand
__global__ void __launch_bounds__(128) percep_pack_rgb_kernel(const float *__restrict__ rgb, int H, int W, Operand dst) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const int64_t HW = (int64_t)H * W, p = (int64_t)y * W + x;
  const float mean[3] = {FAV_MEAN_B, FAV_MEAN_G, FAV_MEAN_R};
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = c < 3 ? __fsub_rn(__fmul_rn(__ldg(rgb + (2 - c) * HW + p), 255.0f), mean[c]) : 0.f;
  const int64_t o = dst.off16(dst.padT + y, 0, dst.padL + x);
  split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
}

// raw conv output -> [ReLU] [max-pool] -> next convolution's operand
__global__ void __launch_bounds__(128) percep_pack_operand_kernel(const float4 *__restrict__ raw, int Cq, int Wp, int Hin, int Win,
                                                                  int relu, PoolSpec pl, Operand dst, int *overflow) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y, cb = blockIdx.z;
  if (x >= dst.W) return;
  float v[8];
  gather8(raw, Cq, Wp, Hin, Win, y, x, cb, relu, pl, v);
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (cb * 8 + i >= dst.C) v[i] = 0.f;
    cnt += out_of_fp16(v[i]);
  }
  const int64_t o = dst.off16(dst.padT + y, cb, dst.padL + x);
  split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
  flush_count(cnt, overflow);
}

// raw conv output -> [ReLU] [max-pool] -> tap [P/8][Cp][8 pixels]: one thread per (8-pixel block, 8-channel block)
__global__ void __launch_bounds__(128) percep_pack_tap_kernel(const float4 *__restrict__ raw, int Cq, int Wp, int Hin, int Win,
                                                              int relu, PoolSpec pl, int C, int Ho, int Wo, int Cp,
                                                              uint4 *__restrict__ hi, uint4 *__restrict__ lo, int *overflow) {
  const int kb = blockIdx.x * 128 + threadIdx.x, cb = blockIdx.y;
  const int64_t P = (int64_t)Ho * Wo;
  if ((int64_t)kb * 8 >= P) return;
  float v[8][8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int64_t p = (int64_t)kb * 8 + q;
    if (p < P) {
      const int y = (int)(p / Wo), x = (int)(p - (int64_t)y * Wo);
      gather8(raw, Cq, Wp, Hin, Win, y, x, cb, relu, pl, v[q]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[q][i] = 0.f;
    }
  }
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = cb * 8 + i;
    if (c >= C) break;
    uint32_t h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      cnt += out_of_fp16(v[2 * q][i]) + out_of_fp16(v[2 * q + 1][i]);
      split_pair(v[2 * q][i], v[2 * q + 1][i], h[q], l[q]);
    }
    const int64_t o = (int64_t)kb * Cp + c;
    hi[o] = make_uint4(h[0], h[1], h[2], h[3]);
    lo[o] = make_uint4(l[0], l[1], l[2], l[3]);
  }
  flush_count(cnt, overflow);
}

__device__ __forceinline__ void join8(uint4 h, uint4 l, float v[8]) {
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __half2float(__ushort_as_half((unsigned short)(hw[i] & 0xffff))) +
               __half2float(__ushort_as_half((unsigned short)(lw[i] & 0xffff)));
    v[2 * i + 1] = __half2float(__ushort_as_half((unsigned short)(hw[i] >> 16))) +
                   __half2float(__ushort_as_half((unsigned short)(lw[i] >> 16)));
  }
}

// fixed-order block reduction of one double per thread (blockDim.x == NT, a power of two); result in thread 0
template <int NT>
__device__ __forceinline__ double block_sum(double v, double *sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

constexpr int kRedThreads = 256, kRedBlocks = 528;

// content loss: sum over the tap of (a - b)^2 (padding is zero in both) -> one double per block
__global__ void __launch_bounds__(kRedThreads) percep_sqdiff_kernel(const uint4 *__restrict__ ah, const uint4 *__restrict__ al,
                                                                    const uint4 *__restrict__ bh, const uint4 *__restrict__ bl,
                                                                    int64_t n16, double *__restrict__ partial) {
  __shared__ double sh[kRedThreads];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kRedThreads + threadIdx.x; i < n16; i += (int64_t)gridDim.x * kRedThreads) {
    float a[8], b[8];
    join8(__ldg(ah + i), __ldg(al + i), a);
    join8(__ldg(bh + i), __ldg(bl + i), b);
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float d = a[k] - b[k];
      t = fmaf(d, d, t);
    }
    s += (double)t;
  }
  const double r = block_sum<kRedThreads>(s, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = r;
}

// out[0] = scale * sum_i p[i] (one block, fixed order)
__global__ void __launch_bounds__(kRedThreads) percep_sum_kernel(const double *__restrict__ p, int n, double scale, double *out) {
  __shared__ double sh[kRedThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) s += p[i];
  const double r = block_sum<kRedThreads>(s, sh);
  if (threadIdx.x == 0) out[0] = scale * r;
}

// out[0] = scale * sum_i (a[i] - t[i])^2 (one block, fixed order): the MSE of the Gram / mean aggregates
__global__ void __launch_bounds__(kRedThreads) percep_vec_sqdiff_kernel(const double *__restrict__ a, const double *__restrict__ t,
                                                                        int n, double scale, double *out) {
  __shared__ double sh[kRedThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) {
    const double d = a[i] - t[i];
    s += d * d;
  }
  const double r = block_sum<kRedThreads>(s, sh);
  if (threadIdx.x == 0) out[0] = scale * r;
}

// style_target_type 'mean' (StyleLoss.lua:18-22: two nn.Mean over the spatial dimensions): one block per channel
__global__ void __launch_bounds__(kRedThreads) percep_chmean_kernel(const uint4 *__restrict__ hi, const uint4 *__restrict__ lo, int Cp,
                                                                    int64_t nkb, double inv_hw, double *__restrict__ out) {
  __shared__ double sh[kRedThreads];
  const int c = blockIdx.x;
  double s = 0.0;
  for (int64_t kb = threadIdx.x; kb < nkb; kb += kRedThreads) {
    float v[8];
    join8(__ldg(hi + kb * Cp + c), __ldg(lo + kb * Cp + c), v);
    s += (double)(((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7])));
  }
  const double r = block_sum<kRedThreads>(s, sh);
  if (threadIdx.x == 0) out[c] = r * inv_hw;
}

// ---- Gram matrix on the tensor cores --------------------------------------------------------------------------------
// CTA = one 64 x 64 tile (row block mt <= column block nt: the upper triangle, G is symmetric) over one contiguous range of
// 128-pixel chunks (split-K).  Warps 0-3: one consumer warpgroup issuing wgmma m64n64k16 (hi*hi + lo*hi + hi*lo per K16 step,
// fp32 accumulators); warp 4: producer, one 1 KB bulk copy per (8-pixel block, operand, hi/lo) into a 3-stage ring.
// Each CTA writes its fp32 partial tile; percep_gram_finish_kernel adds the splits in order, in double.
constexpr int kGramKb = 16;                          // 8-pixel blocks per chunk (128 pixels)
constexpr int kGramStages = 3;
constexpr int kGramFlush = 4;                        // chunks (512 pixels) per fp32 accumulation, then added in double
constexpr int kGramTile16 = kGramKb * 64;            // one 64-channel x 128-pixel fp16 tile, 16-byte units (16 KB)
constexpr int kGramSmem = kGramStages * 4 * kGramTile16 * 16;
constexpr int kGramThreads = 160;

__global__ void __launch_bounds__(kGramThreads, 1) percep_gram_kernel(const uint4 *__restrict__ hi, const uint4 *__restrict__ lo,
                                                                      int Cp, int nchunks, int nsplit, float *__restrict__ part) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t full[kGramStages], empty[kGramStages];
  const int T = Cp / 64;
  int t = blockIdx.x, mt = 0;
  while (t >= T - mt) { t -= T - mt; ++mt; }
  const int nt = mt + t, split = blockIdx.y;
  const int c0 = (int)((int64_t)nchunks * split / nsplit), c1 = (int)((int64_t)nchunks * (split + 1) / nsplit);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kGramStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 4) {
    uint32_t s = 0, ph = 0;
    for (int c = c0; c < c1; ++c) {
      mbar_wait(&empty[s], ph ^ 1);
      if (lane == 0) mbar_arrive_expect_tx(&full[s], 4u * kGramTile16 * 16u);
      __syncwarp();
      uint8_t *st = smem + (size_t)s * 4 * kGramTile16 * 16;
      for (int q = lane; q < 4 * kGramKb; q += 32) {
        const int op = q / kGramKb, kb = q - op * kGramKb;  // op: 0 A hi, 1 A lo, 2 B hi, 3 B lo
        const int row0 = (op < 2 ? mt : nt) * 64;
        const uint4 *src = ((op & 1) ? lo : hi) + ((int64_t)c * kGramKb + kb) * Cp + row0;
        bulk_g2s(st + ((size_t)op * kGramTile16 + kb * 64) * 16, src, 64u * 16u, &full[s]);
      }
      if (++s == kGramStages) { s = 0; ph ^= 1; }
    }
    return;
  }
  // fp32 accumulators cover kGramFlush chunks at a time, then move into double: a 720p relu1_2 split spans ~55 chunks
  // of non-negative products, and one fp32 sum over all of them put the style loss 2.4e-4 off the oracle (H100)
  float acc[32];
  double dacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { acc[i] = 0.f; dacc[i] = 0.0; }
  // descriptor: LBO = 64 x 16 B (next 8-pixel block = next K core matrix), SBO = 8 x 16 B (next 8 channels)
  constexpr uint64_t kDesc = ((uint64_t)8u << 32) | ((uint64_t)64u << 16);
  uint32_t s = 0, ph = 0;
  for (int c = c0; c < c1; ++c) {
    mbar_wait(&full[s], ph);
    const uint32_t base16 = smem_u32(smem + (size_t)s * 4 * kGramTile16 * 16) >> 4;
    uint32_t scale = (c - c0) % kGramFlush ? 1u : 0u;  // the first MMA of a flush block overwrites the accumulators
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kGramKb / 2; ++k) {
      const uint32_t a = base16 + (uint32_t)k * 128u;  // two 8-pixel blocks per K16 step
      const uint64_t ah = kDesc | a, al = kDesc | (a + kGramTile16), bh = kDesc | (a + 2 * kGramTile16),
                     bl = kDesc | (a + 3 * kGramTile16);
      Wgmma<64>::mma(acc, ah, bh, scale);
      Wgmma<64>::mma(acc, al, bh, 1u);
      Wgmma<64>::mma(acc, ah, bl, 1u);
      scale = 1u;
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (threadIdx.x == 0) mbar_arrive(&empty[s]);
    if (++s == kGramStages) { s = 0; ph ^= 1; }
    if ((c - c0) % kGramFlush == kGramFlush - 1 || c == c1 - 1)
#pragma unroll
      for (int i = 0; i < 32; ++i) dacc[i] += (double)acc[i];
  }
  // acc[4i + j]: row 16 w + lane/4 + 8 (j/2), column 8 i + 2 (lane%4) + j%2 (wgmma_f16.cuh)
  float *P = part + (size_t)split * Cp * Cp;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = mt * 64 + 16 * warp + (lane >> 2) + 8 * (j >> 1), col = nt * 64 + 8 * i + 2 * (lane & 3) + (j & 1);
      P[(size_t)r * Cp + col] = (float)dacc[4 * i + j];
    }
}

// G[i][j] = sum over splits (in order, double) / (C H W)  (GramMatrix.lua:47-50); the lower triangle reads the upper tile
__global__ void __launch_bounds__(256) percep_gram_finish_kernel(const float *__restrict__ part, int nsplit, int Cp, int C,
                                                                 double inv_chw, double *__restrict__ G) {
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= C * C) return;
  int a = idx / C, b = idx - (idx / C) * C;
  if (a / 64 > b / 64) { const int tmp = a; a = b; b = tmp; }
  double v = 0.0;
  for (int s = 0; s < nsplit; ++s) v += (double)part[((size_t)s * Cp + a) * Cp + b];
  G[idx] = v * inv_chw;
}

// tap -> fp32 NCHW [C][H][W] (tests, fav_percep_layer_output)
__global__ void __launch_bounds__(256) percep_unpack_tap_kernel(const uint16_t *__restrict__ hi, const uint16_t *__restrict__ lo, int Cp,
                                                                int C, int64_t P, float *__restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y;
  if (p >= P) return;
  const int64_t o = ((p >> 3) * Cp + c) * 8 + (p & 7);
  out[(int64_t)c * P + p] = __half2float(__ushort_as_half(hi[o])) + __half2float(__ushort_as_half(lo[o]));
}

// raw conv output (layout [H][Cq][Wp][4]) -> fp32 NCHW [C][H][W] (tests, fav_percep_conv_output)
__global__ void __launch_bounds__(256) percep_unpack_raw_kernel(const float *__restrict__ raw, int Cq, int Wp, int C, int H, int W,
                                                                float *__restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y;
  if (p >= (int64_t)H * W) return;
  const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
  out[(int64_t)c * H * W + p] = raw[(((int64_t)y * Cq + (c >> 2)) * Wp + x) * 4 + (c & 3)];
}

// ---- backward (fav_percep_forward_backward) ---------------------------------------------------------------------------
// The input gradient of a stride-1 convolution with pad (k-1)/2 is the same convolution geometry over the output gradient, with
// the filters transposed and flipped: it runs on conv_tc_kernel like the forward.  Its operand is the fp16 hi/lo pair, whose
// normal range starts at 6e-5 while the loss gradients sit near 1e-7 and shrink as they flow back, so every gradient operand is
// packed multiplied by a per-tensor power of two that maps its max |g| into [2^14, 2^15).  The factor is exact, so it changes no
// rounding; the kernel that reads the convolution's fp32 output divides it out.  The max lives in device memory.

// 2^k for max |g| (float bits) in [2^(14-k), 2^(15-k)); 1 for an all-zero tensor.  |k| <= 126 keeps 2^k and 2^-k normal.
__device__ __forceinline__ int grad_scale_exp(unsigned maxbits) {
  if (maxbits == 0) return 0;
  const int e = max((int)((maxbits >> 23) & 0xff), 1) - 127;  // floor(log2 max); subnormals as 2^-126
  return min(max(14 - e, -126), 126);
}
__device__ __forceinline__ float grad_scale(unsigned maxbits) { return ldexpf(1.f, grad_scale_exp(maxbits)); }
__device__ __forceinline__ float grad_unscale(unsigned maxbits) { return ldexpf(1.f, -grad_scale_exp(maxbits)); }

// max of |v| over the block -> one atomicMax per warp on the float bits (an order-independent result)
__device__ __forceinline__ void flush_absmax(float m, unsigned *out) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// net-space input [3][H][W] (BGR, 255 x - mean: what PerceptualCriterion:forward receives) -> the first convolution's operand
__global__ void __launch_bounds__(128) percep_pack_net_kernel(const float *__restrict__ in, int H, int W, Operand dst) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const int64_t HW = (int64_t)H * W, p = (int64_t)y * W + x;
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = c < 3 ? __ldg(in + c * HW + p) : 0.f;
  const int64_t o = dst.off16(dst.padT + y, 0, dst.padL + x);
  split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
}

// ContentLoss:updateGradInput (ContentLoss.lua:50-59, MSECriterion): g (+)= strength * 2 (F - F_t) / (C H W), one thread per (pixel, channel)
__global__ void __launch_bounds__(256) percep_content_grad_kernel(const uint16_t *__restrict__ ah, const uint16_t *__restrict__ al,
                                                                  const uint16_t *__restrict__ bh, const uint16_t *__restrict__ bl,
                                                                  int Cp, int64_t P, float coef, int accumulate,
                                                                  float *__restrict__ g) {
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y;
  if (p >= P) return;
  const int64_t o = ((p >> 3) * Cp + c) * 8 + (p & 7);
  const float a = __half2float(__ushort_as_half(ah[o])) + __half2float(__ushort_as_half(al[o]));
  const float b = __half2float(__ushort_as_half(bh[o])) + __half2float(__ushort_as_half(bl[o]));
  const float v = coef * (a - b);
  float *d = g + (int64_t)c * P + p;
  *d = accumulate ? *d + v : v;
}

// StyleLoss 'mean' (two nn.Mean, StyleLoss.lua:57-67): g (+)= strength * 2 (mu_c - t_c) / C / (H W), broadcast over the pixels
__global__ void __launch_bounds__(256) percep_mean_grad_kernel(const double *__restrict__ mu, const double *__restrict__ t, int64_t P,
                                                               double coef, int accumulate, float *__restrict__ g) {
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y;
  if (p >= P) return;
  const float v = (float)(coef * (mu[c] - t[c]));
  float *d = g + (int64_t)c * P + p;
  *d = accumulate ? *d + v : v;
}

// D = strength * 4 (G - T) / (C^2 C H W), formed in double and rounded once (G and T are symmetric, so is D)
__global__ void __launch_bounds__(256) percep_gram_diff_kernel(const double *__restrict__ G, const double *__restrict__ T, int n,
                                                               double coef, float *__restrict__ D) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) D[i] = (float)(coef * (G[i] - T[i]));
}

// GramMatrix:updateGradInput (GramMatrix.lua:54-78) after StyleLoss: g[c][p] (+)= sum_j D[c][j] F[j][p], F the tap (hi + lo).
// CTA tile: 64 channels x 128 pixels, K = 16 channels per shared-memory step; thread: 4 channels x 8 pixels (p = tp + 16 i), fp32.
// Every output element is written by one thread, with a fixed summation order.
constexpr int kGbM = 64, kGbN = 128, kGbK = 16;
__global__ void __launch_bounds__(256) percep_gram_grad_kernel(const float *__restrict__ D, const uint4 *__restrict__ hi,
                                                               const uint4 *__restrict__ lo, int C, int Cp, int64_t P, int accumulate,
                                                               float *__restrict__ g) {
  __shared__ float As[kGbK][kGbM];
  __shared__ float Bs[kGbK][kGbN];
  const int t = threadIdx.x, tc = t >> 4, tp = t & 15;
  const int c0 = blockIdx.y * kGbM;
  const int64_t p0 = (int64_t)blockIdx.x * kGbN;
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int j0 = 0; j0 < C; j0 += kGbK) {
    {  // A: D[j0 + k][c0 + 4 q + i] (= D[c][j], symmetric)
      const int k = t >> 4, q = t & 15, j = j0 + k;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + 4 * q + i;
        As[k][4 * q + i] = (j < C && c < C) ? __ldg(D + (int64_t)j * C + c) : 0.f;
      }
    }
    {  // B: F[j0 + k][p0 + 8 b .. + 8]: one 16-byte hi / lo unit of the tap layout [P/8][Cp][8]
      const int k = t >> 4, b = t & 15, j = j0 + k;
      float v[8];
      const int64_t kb = (p0 >> 3) + b;
      if (j < Cp && (kb << 3) < P) {
        join8(__ldg(hi + kb * Cp + j), __ldg(lo + kb * Cp + j), v);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) Bs[k][8 * b + i] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kGbK; ++k) {
      float a[4], b[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][4 * tc + i];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = Bs[k][tp + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + 4 * tc + i;
    if (c >= C) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t p = p0 + tp + 16 * j;
      if (p >= P) continue;
      float *d = g + (int64_t)c * P + p;
      *d = accumulate ? *d + acc[i][j] : acc[i][j];
    }
  }
}

// One stage of the backward pass: the gradient at the raw output of conv s (bias included), from
//  - the gradient at the input of conv s + 1 (the fp32 output of its input-gradient convolution, scaled by 2^k), and
//  - the gradient of every loss layer of this stage (planar fp32 [C][H][W] at the loss layer's own size),
// each passed back through the modules between conv s and its place: max-pooling as a gather (each pixel sums the windows whose
// first maximum in row-major order it is; no atomics), ReLU as the mask raw > 0 (nn.ReLU(true): its input is its output, and
// max-pooling commutes with the ReLU, so pooled-then-rectified terms use the same mask).  One thread per (pixel, channel quad).
constexpr int kMaxStageTerms = 8;
struct BwdTerm {
  const float *g;  // planar [C][H][W]; null for the next-stage term, which reads `nxt`
  int H, W, relu, pool;
};
struct BwdStage {
  const float4 *raw;
  int C, Cq, Wp, H, W;
  PoolSpec pool;          // the stage's max-pooling (pooled terms)
  const float4 *nxt;      // next-stage term: raw layout, nxt_Wp pitch, the same channel quads; null at the deepest stage
  int nxt_Wp;
  const unsigned *nxt_max;
  int nt;
  BwdTerm t[kMaxStageTerms];
  float4 *out;            // raw layout (Cq, Wp)
  unsigned *out_max;
};

__device__ __forceinline__ void term_at(const BwdStage &s, const BwdTerm &tm, int cq, int y, int x, float inv, float v[4]) {
  if (!tm.g) {
    const float4 a = __ldg(s.nxt + ((int64_t)y * s.Cq + cq) * s.nxt_Wp + x);
    v[0] = a.x * inv; v[1] = a.y * inv; v[2] = a.z * inv; v[3] = a.w * inv;
    return;
  }
  const int64_t HW = (int64_t)tm.H * tm.W, p = (int64_t)y * tm.W + x;
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = 4 * cq + i < s.C ? __ldg(tm.g + (4 * cq + i) * HW + p) : 0.f;
}

__global__ void __launch_bounds__(128) percep_bwd_stage_kernel(const BwdStage s) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y, cq = blockIdx.z;
  float m = 0.f;
  if (x < s.W) {
    const float inv = s.nxt ? grad_unscale(*s.nxt_max) : 0.f;
    float ap[4] = {0.f, 0.f, 0.f, 0.f}, ar[4] = {0.f, 0.f, 0.f, 0.f};  // unmasked / ReLU-masked sums
    bool pooled = false;
    for (int k = 0; k < s.nt; ++k) {
      const BwdTerm &tm = s.t[k];
      if (tm.pool) { pooled = true; continue; }
      float v[4];
      term_at(s, tm, cq, y, x, inv, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) (tm.relu ? ar : ap)[i] += v[i];
    }
    if (pooled) {
      const PoolSpec &pl = s.pool;
      const int oy0 = max(0, (y + pl.ph - pl.kh + pl.sh) / pl.sh), oy1 = (y + pl.ph) / pl.sh;
      const int ox0 = max(0, (x + pl.pw - pl.kw + pl.sw) / pl.sw), ox1 = (x + pl.pw) / pl.sw;
      // the pooled grid: every pooled term has the same extents (BwdTerm H / W)
      int Ho = 0, Wo = 0;
      for (int k = 0; k < s.nt; ++k)
        if (s.t[k].pool) { Ho = s.t[k].H; Wo = s.t[k].W; break; }
      for (int oy = oy0; oy <= min(oy1, Ho - 1); ++oy)
        for (int ox = ox0; ox <= min(ox1, Wo - 1); ++ox) {
          const int hs = oy * pl.sh - pl.ph, ws = ox * pl.sw - pl.pw;
          const int he = min(hs + pl.kh, s.H), we = min(ws + pl.kw, s.W);
          float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
          int bi[4] = {-1, -1, -1, -1};
          for (int iy = max(hs, 0); iy < he; ++iy)
            for (int ix = max(ws, 0); ix < we; ++ix) {
              const float4 a = __ldg(s.raw + ((int64_t)iy * s.Cq + cq) * s.Wp + ix);
              const float av[4] = {a.x, a.y, a.z, a.w};
              const int id = iy * s.W + ix;
#pragma unroll
              for (int i = 0; i < 4; ++i)
                if (av[i] > best[i]) { best[i] = av[i]; bi[i] = id; }
            }
          const int self = y * s.W + x;
          if (bi[0] != self && bi[1] != self && bi[2] != self && bi[3] != self) continue;
          for (int k = 0; k < s.nt; ++k) {
            const BwdTerm &tm = s.t[k];
            if (!tm.pool) continue;
            float v[4];
            term_at(s, tm, cq, oy, ox, inv, v);
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if (bi[i] == self) (tm.relu ? ar : ap)[i] += v[i];
          }
        }
    }
    const float4 r = __ldg(s.raw + ((int64_t)y * s.Cq + cq) * s.Wp + x);
    const float rv[4] = {r.x, r.y, r.z, r.w};
    float g[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      g[i] = 4 * cq + i < s.C ? ap[i] + (rv[i] > 0.f ? ar[i] : 0.f) : 0.f;
      m = fmaxf(m, fabsf(g[i]));
    }
    s.out[((int64_t)y * s.Cq + cq) * s.Wp + x] = make_float4(g[0], g[1], g[2], g[3]);
  }
  flush_absmax(m, s.out_max);
}

// gradient (raw layout) x 2^k -> the input-gradient convolution's operand (fp16 hi / lo, zero border kept)
__global__ void __launch_bounds__(128) percep_bwd_pack_kernel(const float4 *__restrict__ g, int Cq, int Wp, const unsigned *gmax,
                                                              Operand dst) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y, cb = blockIdx.z;
  if (x >= dst.W) return;
  const float sc = grad_scale(*gmax);
  const float4 a = __ldg(g + ((int64_t)y * Cq + 2 * cb) * Wp + x);
  const float4 b = 2 * cb + 1 < Cq ? __ldg(g + ((int64_t)y * Cq + 2 * cb + 1) * Wp + x) : make_float4(0.f, 0.f, 0.f, 0.f);
  float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = cb * 8 + i < dst.C ? v[i] * sc : 0.f;
  const int64_t o = dst.off16(dst.padT + y, cb, dst.padL + x);
  split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
}

// the first convolution's input gradient (raw layout, 2^k scaled) -> grad_input [3][H][W] fp32
__global__ void __launch_bounds__(256) percep_grad_input_kernel(const float4 *__restrict__ d, int Wp, const unsigned *gmax, int H, int W,
                                                                float *__restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (p >= (int64_t)H * W) return;
  const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
  const float inv = grad_unscale(*gmax);
  const float4 a = __ldg(d + (int64_t)y * Wp + x);  // Cq = 1
  const int64_t HW = (int64_t)H * W;
  out[p] = a.x * inv;
  out[HW + p] = a.y * inv;
  out[2 * HW + p] = a.z * inv;
}

// ---- pixel loss and TotalVariation gradients (train_video.lua:117-126,354-366; TotalVariation.lua:19-35) -------------
// pixel_crit:forward / backward(out2 .* cert, prev_warped_masked): per-element loss terms and d loss / d (out2 .* cert), added to
// grad_accum WITHOUT the certainty factor (train_video.lua:357-364 adds the criterion's gradInput as it is).  type 0 L2 (MSE),
// 1 L1 (AbsCriterion), 2 SmoothL1; sizeAverage over N*3*H*W (norm: the criterion's fp32 2/n or 1/n), then x weight as
// grad_out:add(weight, grad_pix).  Per-block loss partials in double, summed in a fixed order.
__global__ void __launch_bounds__(kRedThreads) fav_pixel_loss_grad_kernel(const float *__restrict__ out2, const float *__restrict__ prev,
                                                                          const float *__restrict__ cert, int64_t HW, int64_t n, int type,
                                                                          float norm, float weight, float *__restrict__ acc,
                                                                          double *__restrict__ partial) {
  __shared__ double sh[kRedThreads];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kRedThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kRedThreads) {
    const int64_t img = i / (3 * HW), pix = (i - img * 3 * HW) % HW;
    const float a = __fmul_rn(out2[i], __ldg(cert + img * HW + pix));
    const float d = __fsub_rn(a, prev[i]);
    double l;
    float g;
    if (type == 0) { l = (double)d * d; g = __fmul_rn(norm, d); }
    else if (type == 1) { l = fabs((double)d); g = d >= 0.f ? norm : -norm; }
    else {
      const double z = fabs((double)d);
      l = z < 1.0 ? 0.5 * z * z : z - 0.5;
      g = d < -1.f ? -norm : (d > 1.f ? norm : __fmul_rn(norm, d));
    }
    s += l;
    acc[i] = __fadd_rn(acc[i], __fmul_rn(weight, g));
  }
  const double r = block_sum<kRedThreads>(s, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = r;
}

// TotalVariation:updateGradInput with its {1,-2} ranges, as a gather, in the module's fp32 order: diffs on the (H-1) x (W-1)
// corner, added into zero, then strength x, then added to grad_accum (the module's gradOutput)
__global__ void __launch_bounds__(256) fav_tv_grad_kernel(const float *__restrict__ x, int64_t planes, int H, int W, float strength,
                                                          float *__restrict__ acc) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int64_t HW = (int64_t)H * W;
  if (i >= planes * HW) return;
  const int64_t pl = i / HW;
  const int p = (int)(i - pl * HW), yy = p / W, xx = p - yy * W;
  const float *X = x + pl * HW;
  auto at = [&](int y, int xc) { return X[(int64_t)y * W + xc]; };
  float t = 0.f;
  if (yy < H - 1 && xx < W - 1) {
    t = t + (at(yy, xx) - at(yy, xx + 1));
    t = t + (at(yy, xx) - at(yy + 1, xx));
  }
  if (yy < H - 1 && xx >= 1) t = t - (at(yy, xx - 1) - at(yy, xx));
  if (yy >= 1 && xx < W - 1) t = t - (at(yy - 1, xx) - at(yy, xx));
  acc[i] = __fadd_rn(acc[i], __fmul_rn(t, strength));
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
struct PModule {
  int kind = 0;  // 0 conv, 1 ReLU, 2 max-pool
  int cin = 0, cout = 0, k = 0, stride = 1, pad = 0;
  PoolSpec pool{0, 0, 0, 0, 0, 0, 0};
  int ceil_mode = 0;
};

struct PConv {
  int module = 0;  // 1-based module index
  int cin = 0, cout = 0, k = 0, stride = 1, pad = 0;
  std::vector<float> w, b;
  bool set = false;
  std::vector<ConvDef> blocks;        // one per 128-channel N block
  std::vector<float *> d_bias;        // per block, Npad entries
  // input gradient (fav_percep_forward_backward): a cout -> cin convolution with the flipped, transposed filters and zero
  // bias, one ConvDef per 128-channel N block of cin; packed on the first backward call
  std::vector<ConvDef> dblocks;
  float *d_zero = nullptr;            // kMaxNBlock zero biases
};

struct PTapSpec {  // a loss layer's feature map: (relu, pool) applied to the raw output of conv `stage`
  int index = 0, stage = 0, relu = 0;
  PoolSpec pool{0, 0, 0, 0, 0, 0, 0};
  int ceil_mode = 0;
  bool content = false;
};

struct PStageSpec {  // how the input of conv s + 1 is made from the raw output of conv s
  int relu = 0;
  PoolSpec pool{0, 0, 0, 0, 0, 0, 0};
  int ceil_mode = 0;
};

struct PTap {
  int C = 0, Cp = 0, H = 0, W = 0;
  int64_t nkb = 0;  // 8-pixel blocks, padded to whole Gram chunks
  uint4 *hi = nullptr, *lo = nullptr;
};

struct PPlan {
  int H = 0, W = 0;
  std::vector<Operand> in;             // input operand of every conv
  std::vector<RawTensor> raw;          // output geometry of every conv (all share one buffer)
  std::vector<std::vector<ConvJob>> jobs;
  std::vector<PTap> taps[2];           // [pass][tap]: pass 0 = content target forward, 1 = the evaluated image
  float *gram_part = nullptr;
  size_t gram_part_floats = 0;
  double *red = nullptr;               // reduction partials
  int *overflow = nullptr;
  // backward plans only (build_pplan retain): every raw above has its own buffer, and the gradient buffers
  std::vector<Operand> gop;            // [conv s]: operand of its input-gradient convolution (output gradient x 2^k)
  std::vector<RawTensor> gin;          // [conv s]: that convolution's fp32 output, the gradient at conv s's input (one buffer)
  std::vector<std::vector<ConvJob>> djobs;
  float *gbuf = nullptr;               // one stage's output gradient, raw layout
  std::vector<float *> tgrad;          // [tap]: gradient of the loss layers there, planar [C][H][W]
  float *gram_d = nullptr;             // C x C: strength * 4 (G - T) / (C^2 C H W) of one style layer
  unsigned *gmax = nullptr;            // [conv s]: max |gradient| at its output (float bits)
  std::vector<void *> allocs;
  ~PPlan() {
    for (void *p : allocs) cudaFree(p);
  }
};

static int pool_out(int n, int k, int s, int p, int ceil_mode) {
  // SpatialMaxPooling (THNN): ceil or floor, then "the last pooling starts inside the image" when padded
  int o = ceil_mode ? (int)std::ceil((double)(n - k + 2 * p) / s) + 1 : (int)std::floor((double)(n - k + 2 * p) / s) + 1;
  if (p > 0 && (o - 1) * s >= n + p) --o;
  return o;
}

}  // namespace fav

using namespace fav;

struct fav_percep {
  std::vector<PModule> mods;
  std::vector<PConv> convs;
  std::vector<PStageSpec> next;   // [conv s]: how conv s + 1's input is made
  std::vector<PTapSpec> taps;     // distinct loss layer indices, ascending
  std::vector<int> content_tap, style_tap;
  std::vector<double> content_w, style_w;
  int agg = 0;                    // 0 gram, 1 mean
  int last_content_stage = -1;
  bool finalized = false;
  bool has_target = false;
  int num_sms = 132;
  int bwd_refuse = 0;             // first convolution module whose input gradient is not the same-geometry convolution
  bool bwd_ready = false;         // dblocks packed
  std::map<std::pair<int, int>, std::unique_ptr<PPlan>> plans;
  std::map<std::pair<int, int>, std::unique_ptr<PPlan>> bplans;  // fav_percep_forward_backward: raw outputs kept
  PPlan *last_plan = nullptr;
  bool last_backward = false;     // last_plan is a backward plan (fav_percep_conv_output)
  std::vector<double *> target, stat;  // per style layer: aggregate of the style image / of the last evaluated image
  double *d_losses = nullptr;          // [n_content + n_style]
  std::vector<void *> allocs;
  ~fav_percep() {
    plans.clear();
    bplans.clear();
    for (void *p : allocs) cudaFree(p);
  }
};

namespace fav {

static int p_alloc(std::vector<void *> &allocs, void **out, size_t bytes) {
  FAV_TRY(check_cuda(cudaMalloc(out, std::max<size_t>(bytes, 16)), "cudaMalloc(percep)"));
  allocs.push_back(*out);
  return check_cuda(cudaMemset(*out, 0, std::max<size_t>(bytes, 16)), "cudaMemset(percep)");
}

static int tap_size(const PTapSpec &t, const std::vector<RawTensor> &raw, int *H, int *W) {
  const RawTensor &r = raw[t.stage];
  *H = r.H; *W = r.W;
  if (t.pool.on) {
    *H = pool_out(r.H, t.pool.kh, t.pool.sh, t.pool.ph, t.ceil_mode);
    *W = pool_out(r.W, t.pool.kw, t.pool.sw, t.pool.pw, t.ceil_mode);
  }
  if (*H < 1 || *W < 1) {
    set_error("loss network: layer %d has an empty output at this image size", t.index);
    return FAV_ERR_INVALID;
  }
  return FAV_OK;
}

static int build_backward(fav_percep *P, PPlan &pl);

// retain: a backward plan (P->bplans) -- every convolution's raw output in its own buffer, plus the gradient buffers
static int build_pplan(fav_percep *P, int H, int W, PPlan **out, bool retain = false) {
  auto &plans = retain ? P->bplans : P->plans;
  auto key = std::make_pair(H, W);
  auto it = plans.find(key);
  if (it != plans.end()) { *out = it->second.get(); return FAV_OK; }
  FAV_REQUIRE(H >= 1 && W >= 1, "fav_percep: bad image size %dx%d", W, H);
  std::unique_ptr<PPlan> pl(new PPlan());
  pl->H = H; pl->W = W;
  const int ns = (int)P->convs.size();
  // sizes
  int h = H, w = W;
  size_t raw_max = 0;
  for (int s = 0; s < ns; ++s) {
    const PConv &pc = P->convs[s];
    Operand o = operand_geometry(pc.cin, h, w, &pc.blocks[0]);
    pl->in.push_back(o);
    int ho, wo;
    conv_out_size(pc.blocks[0], h, w, &ho, &wo);
    if (ho < 1 || wo < 1) {
      set_error("loss network: module %d (convolution) has an empty output at %dx%d", pc.module, W, H);
      return FAV_ERR_INVALID;
    }
    RawTensor r;
    r.C = pc.cout; r.Cq = round_up(pc.cout, 4) / 4; r.H = ho; r.W = wo; r.Hp = ho + 2; r.Wp = round_up(wo, kTileM);
    raw_max = std::max(raw_max, (size_t)r.Hp * r.Cq * r.Wp * 4);
    pl->raw.push_back(r);
    h = ho; w = wo;
    if (s + 1 < ns) {
      const PStageSpec &nx = P->next[s];
      if (nx.pool.on) {
        h = pool_out(ho, nx.pool.kh, nx.pool.sh, nx.pool.ph, nx.ceil_mode);
        w = pool_out(wo, nx.pool.kw, nx.pool.sw, nx.pool.pw, nx.ceil_mode);
        if (h < 1 || w < 1) { set_error("loss network: max-pooling before module %d empties the map", P->convs[s + 1].module); return FAV_ERR_INVALID; }
      }
    }
  }
  if (retain) {
    for (RawTensor &r : pl->raw) FAV_TRY(p_alloc(pl->allocs, (void **)&r.p, (size_t)r.Hp * r.Cq * r.Wp * 4 * sizeof(float) + 4096));
  } else {
    float *raw_buf = nullptr;
    FAV_TRY(p_alloc(pl->allocs, (void **)&raw_buf, raw_max * sizeof(float) + 4096));
    for (RawTensor &r : pl->raw) r.p = raw_buf;
  }
  for (int s = 0; s < ns; ++s) {
    Operand &o = pl->in[s];
    FAV_TRY(p_alloc(pl->allocs, (void **)&o.hi, o.elems16 * 16));
    FAV_TRY(p_alloc(pl->allocs, (void **)&o.lo, o.elems16 * 16));
  }
  // conv jobs: one per N block
  pl->jobs.resize(ns);
  for (int s = 0; s < ns; ++s) {
    PConv &pc = P->convs[s];
    const RawTensor &r = pl->raw[s];
    for (size_t b = 0; b < pc.blocks.size(); ++b) {
      ConvDef &c = pc.blocks[b];
      ConvJob j;
      if (fill_conv_job(c, c.phases[0], pl->in[s], j) != FAV_OK) {
        const std::string why = fav_last_error();
        set_error("loss network: module %d (convolution): %s", pc.module, why.c_str());
        return FAV_ERR_UNSUPPORTED;
      }
      j.b = c.phases[0].d_b_tc; j.bias = pc.d_bias[b];
      j.raw = r.p + conv_nblock_raw_offset((int)b, r.Wp); j.raw_Cq = r.Cq; j.raw_Wp = r.Wp;
      j.final_mode = 0;
      conv_tc_choose_slots(j);
      if (conv_tc_smem_bytes(j) > 227 * 1024 || (!j.b_resident && j.b_slots < 2)) {
        set_error("loss network: module %d (convolution): shared memory budget exceeded", pc.module);
        return FAV_ERR_UNSUPPORTED;
      }
      pl->jobs[s].push_back(j);
    }
  }
  // taps (pass 0: content layers only)
  size_t part_max = 16;
  for (int pass = 0; pass < 2; ++pass)
    for (const PTapSpec &t : P->taps) {
      PTap tp;
      if (pass == 1 || t.content) {
        FAV_TRY(tap_size(t, pl->raw, &tp.H, &tp.W));
        tp.C = P->convs[t.stage].cout; tp.Cp = round_up(tp.C, 64);
        const int64_t nkb = ceil_div64((int64_t)tp.H * tp.W, 8);
        tp.nkb = ceil_div64(nkb, kGramKb) * kGramKb;  // whole 128-pixel Gram chunks, zero padded
        FAV_TRY(p_alloc(pl->allocs, (void **)&tp.hi, (size_t)tp.nkb * tp.Cp * 16));
        FAV_TRY(p_alloc(pl->allocs, (void **)&tp.lo, (size_t)tp.nkb * tp.Cp * 16));
        const int T = tp.Cp / 64, ntri = T * (T + 1) / 2;
        const int nchunks = (int)(tp.nkb / kGramKb);
        const int nsplit = std::max(1, std::min(nchunks, P->num_sms / ntri));
        part_max = std::max(part_max, (size_t)nsplit * tp.Cp * tp.Cp);
      }
      pl->taps[pass].push_back(tp);
    }
  FAV_TRY(p_alloc(pl->allocs, (void **)&pl->gram_part, part_max * sizeof(float)));
  pl->gram_part_floats = part_max;
  FAV_TRY(p_alloc(pl->allocs, (void **)&pl->red, (size_t)kRedBlocks * sizeof(double)));
  FAV_TRY(p_alloc(pl->allocs, (void **)&pl->overflow, sizeof(int)));
  if (retain) FAV_TRY(build_backward(P, *pl));
  *out = pl.get();
  plans[key] = std::move(pl);
  return FAV_OK;
}

// the gradient side of a backward plan: per conv s the operand of its input-gradient convolution (at conv s's output size, the
// padding of the dgrad ConvDef) and that convolution's jobs writing into one shared fp32 buffer; per tap a planar loss gradient
static int build_backward(fav_percep *P, PPlan &pl) {
  const int ns = (int)P->convs.size();
  size_t graw = 16, draw = 16;
  pl.gop.resize(ns); pl.gin.resize(ns); pl.djobs.resize(ns);
  for (int s = 0; s < ns; ++s) {
    const PConv &pc = P->convs[s];
    const RawTensor &r = pl.raw[s];
    Operand &o = pl.gop[s];
    o = operand_geometry(pc.cout, r.H, r.W, &pc.dblocks[0]);
    FAV_TRY(p_alloc(pl.allocs, (void **)&o.hi, o.elems16 * 16));
    FAV_TRY(p_alloc(pl.allocs, (void **)&o.lo, o.elems16 * 16));
    RawTensor &d = pl.gin[s];
    d.C = pc.cin; d.Cq = round_up(pc.cin, 4) / 4; d.H = pl.in[s].H; d.W = pl.in[s].W; d.Hp = d.H + 2; d.Wp = round_up(d.W, kTileM);
    graw = std::max(graw, (size_t)r.Hp * r.Cq * r.Wp * 4);
    draw = std::max(draw, (size_t)d.Hp * d.Cq * d.Wp * 4);
  }
  float *dbuf = nullptr;
  FAV_TRY(p_alloc(pl.allocs, (void **)&pl.gbuf, graw * sizeof(float) + 4096));
  FAV_TRY(p_alloc(pl.allocs, (void **)&dbuf, draw * sizeof(float) + 4096));
  for (int s = 0; s < ns; ++s) {
    PConv &pc = P->convs[s];
    RawTensor &d = pl.gin[s];
    d.p = dbuf;
    for (size_t b = 0; b < pc.dblocks.size(); ++b) {
      ConvDef &c = pc.dblocks[b];
      ConvJob j;
      int ho, wo;
      conv_out_size(c, pl.gop[s].H, pl.gop[s].W, &ho, &wo);
      if (ho != d.H || wo != d.W || fill_conv_job(c, c.phases[0], pl.gop[s], j) != FAV_OK) {
        set_error("loss network: module %d (convolution): its input gradient has no tensor-core plan", pc.module);
        return FAV_ERR_UNSUPPORTED;
      }
      j.b = c.phases[0].d_b_tc; j.bias = pc.d_zero;
      j.raw = d.p + conv_nblock_raw_offset((int)b, d.Wp); j.raw_Cq = d.Cq; j.raw_Wp = d.Wp;
      j.final_mode = 0;
      conv_tc_choose_slots(j);
      if (conv_tc_smem_bytes(j) > 227 * 1024 || (!j.b_resident && j.b_slots < 2)) {
        set_error("loss network: module %d (convolution): input gradient exceeds the shared memory budget", pc.module);
        return FAV_ERR_UNSUPPORTED;
      }
      pl.djobs[s].push_back(j);
    }
  }
  size_t dmax = 16;
  for (const PTap &tp : pl.taps[1]) {
    float *g = nullptr;
    FAV_TRY(p_alloc(pl.allocs, (void **)&g, (size_t)tp.C * tp.H * tp.W * sizeof(float)));
    pl.tgrad.push_back(g);
    dmax = std::max(dmax, (size_t)tp.C * tp.C);
  }
  FAV_TRY(p_alloc(pl.allocs, (void **)&pl.gram_d, dmax * sizeof(float)));
  FAV_TRY(p_alloc(pl.allocs, (void **)&pl.gmax, (size_t)ns * sizeof(unsigned)));
  return FAV_OK;
}

static int launch_pack_tap(const RawTensor &r, const PTapSpec &t, const PTap &tp, int *overflow, cudaStream_t st) {
  dim3 grid((unsigned)ceil_div64(ceil_div64((int64_t)tp.H * tp.W, 8), 128), (unsigned)ceil_div(tp.C, 8));
  percep_pack_tap_kernel<<<grid, 128, 0, st>>>(reinterpret_cast<const float4 *>(r.p), r.Cq, r.Wp, r.H, r.W, t.relu, t.pool, tp.C,
                                               tp.H, tp.W, tp.Cp, tp.hi, tp.lo, overflow);
  return post_launch("percep_pack_tap");
}

// one forward of the loss network: pass 0 stops after the deepest content layer and keeps the content taps only.
// img: RGB in [0,1] (the VGG preprocess fused into the first pack), or, net_space, the preprocessed BGR image itself
static int run_pass(fav_percep *P, PPlan &pl, const float *img, int pass, cudaStream_t st, bool net_space = false) {
  const int ns = (int)P->convs.size();
  const int last = pass == 0 ? P->last_content_stage : ns - 1;
  {
    const Operand &o = pl.in[0];
    if (net_space) {
      percep_pack_net_kernel<<<dim3(ceil_div(pl.W, 128), pl.H), 128, 0, st>>>(img, pl.H, pl.W, o);
      FAV_TRY(post_launch("percep_pack_net"));
    } else {
      percep_pack_rgb_kernel<<<dim3(ceil_div(pl.W, 128), pl.H), 128, 0, st>>>(img, pl.H, pl.W, o);
      FAV_TRY(post_launch("percep_pack_rgb"));
    }
  }
  for (int s = 0; s <= last; ++s) {
    for (const ConvJob &j : pl.jobs[s]) FAV_TRY(launch_conv_tc(j, P->num_sms, st));
    const RawTensor &r = pl.raw[s];
    for (size_t t = 0; t < P->taps.size(); ++t) {
      const PTapSpec &ts = P->taps[t];
      if (ts.stage != s || (pass == 0 && !ts.content)) continue;
      FAV_TRY(launch_pack_tap(r, ts, pl.taps[pass][t], pl.overflow, st));
    }
    if (s < last) {
      const PStageSpec &nx = P->next[s];
      const Operand &o = pl.in[s + 1];
      percep_pack_operand_kernel<<<dim3(ceil_div(o.W, 128), o.H, o.Cb), 128, 0, st>>>(
          reinterpret_cast<const float4 *>(r.p), r.Cq, r.Wp, r.H, r.W, nx.relu, nx.pool, o, pl.overflow);
      FAV_TRY(post_launch("percep_pack_operand"));
    }
  }
  return FAV_OK;
}

// aggregate of a style layer's tap (Gram matrix or per-channel means) -> out (double)
static int aggregate(fav_percep *P, PPlan &pl, const PTap &tp, double *out, cudaStream_t st) {
  if (P->agg == 1) {
    percep_chmean_kernel<<<tp.C, kRedThreads, 0, st>>>(tp.hi, tp.lo, tp.Cp, tp.nkb, 1.0 / ((double)tp.H * tp.W), out);
    return post_launch("percep_chmean");
  }
  const int T = tp.Cp / 64, ntri = T * (T + 1) / 2, nchunks = (int)(tp.nkb / kGramKb);
  const int nsplit = std::max(1, std::min(nchunks, P->num_sms / ntri));
  // the > 48 KB shared-memory opt-in is per device: set before every launch (a cheap host call, not a launch)
  FAV_TRY(check_cuda(cudaFuncSetAttribute(percep_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGramSmem),
                     "cudaFuncSetAttribute(percep_gram)"));
  percep_gram_kernel<<<dim3(ntri, nsplit), kGramThreads, kGramSmem, st>>>(tp.hi, tp.lo, tp.Cp, nchunks, nsplit, pl.gram_part);
  FAV_TRY(post_launch("percep_gram"));
  percep_gram_finish_kernel<<<ceil_div(tp.C * tp.C, 256), 256, 0, st>>>(pl.gram_part, nsplit, tp.Cp, tp.C,
                                                                        1.0 / ((double)tp.C * tp.H * tp.W), out);
  return post_launch("percep_gram_finish");
}

static int agg_len(const fav_percep *P, int C) { return P->agg == 1 ? C : C * C; }

static int check_overflow(PPlan &pl, cudaStream_t st) {
  int n = 0;
  FAV_TRY(check_cuda(cudaMemcpyAsync(&n, pl.overflow, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync(overflow)"));
  FAV_TRY(check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize(percep)"));
  if (n) {
    set_error("loss network: %d activation values exceed the fp16 operand range (|x| > 65504); the losses would be computed "
              "from clamped features", n);
    return FAV_ERR_UNSUPPORTED;
  }
  return FAV_OK;
}

// MSE of every loss layer after the two passes -> P->d_losses (content layers, then style layers)
static int launch_losses(fav_percep *p, PPlan &pl, cudaStream_t st) {
  const size_t nc = p->content_tap.size(), nsty = p->style_tap.size();
  for (size_t k = 0; k < nc; ++k) {  // nn.MSECriterion: mean over C*H*W
    const PTap &a = pl.taps[1][p->content_tap[k]], &b = pl.taps[0][p->content_tap[k]];
    percep_sqdiff_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(a.hi, a.lo, b.hi, b.lo, a.nkb * a.Cp, pl.red);
    FAV_TRY(post_launch("percep_sqdiff"));
    percep_sum_kernel<<<1, kRedThreads, 0, st>>>(pl.red, kRedBlocks, 1.0 / ((double)a.C * a.H * a.W), p->d_losses + k);
    FAV_TRY(post_launch("percep_sum"));
  }
  for (size_t k = 0; k < nsty; ++k) {  // nn.MSECriterion over the C x C Gram matrix (or the C means)
    const PTap &a = pl.taps[1][p->style_tap[k]];
    FAV_TRY(aggregate(p, pl, a, p->stat[k], st));
    const int n = agg_len(p, a.C);
    percep_vec_sqdiff_kernel<<<1, kRedThreads, 0, st>>>(p->stat[k], p->target[k], n, 1.0 / n, p->d_losses + nc + k);
    FAV_TRY(post_launch("percep_vec_sqdiff"));
  }
  return FAV_OK;
}

// P->d_losses -> host (synchronises), the overflow check, strength * MSE per layer and the two totals in layer order
// (PerceptualCriterion.lua:141-152)
static int finish_losses(fav_percep *p, PPlan &pl, cudaStream_t st, double *content_loss, double *style_loss, double *layer_losses) {
  const size_t nc = p->content_tap.size(), nsty = p->style_tap.size();
  std::vector<double> mse(nc + nsty + 1, 0.0);
  FAV_TRY(check_cuda(cudaMemcpyAsync(mse.data(), p->d_losses, mse.size() * sizeof(double), cudaMemcpyDeviceToHost, st),
                     "cudaMemcpyAsync(losses)"));
  FAV_TRY(check_overflow(pl, st));
  double tc = 0.0, ts = 0.0;
  for (size_t k = 0; k < nc; ++k) tc += p->content_w[k] * mse[k];
  for (size_t k = 0; k < nsty; ++k) ts += p->style_w[k] * mse[nc + k];
  if (layer_losses) {
    for (size_t k = 0; k < nc; ++k) layer_losses[k] = p->content_w[k] * mse[k];
    for (size_t k = 0; k < nsty; ++k) layer_losses[nc + k] = p->style_w[k] * mse[nc + k];
  }
  *content_loss = tc;
  *style_loss = ts;
  return FAV_OK;
}

// host-only: the first convolution whose input gradient is not a same-geometry convolution (stride 1, pad (k-1)/2), 0 if none
static int bwd_unsupported_module(const fav_percep *P) {
  for (const PConv &pc : P->convs)
    if (pc.stride != 1 || pc.pad != (pc.k - 1) / 2) return pc.module;
  return 0;
}

// host-only: the first stage with more gradient terms than percep_bwd_stage_kernel takes (its loss layers, plus the next stage's
// input gradient), as the module index of its convolution; 0 if none
static int bwd_crowded_stage(const fav_percep *P) {
  const int ns = (int)P->convs.size();
  for (int s = 0; s < ns; ++s) {
    int nt = s + 1 < ns;
    for (const PTapSpec &ts : P->taps) nt += ts.stage == s;
    if (nt > kMaxStageTerms) return P->convs[s].module;
  }
  return 0;
}

// the input-gradient convolutions: W'[ci][co][ky][kx] = W[co][ci][k-1-ky][k-1-kx], a [cin][cout][k][k] tensor read as the
// weights of a cout -> cin convolution, packed per 128-channel N block of cin like the forward's
static int prepare_backward(fav_percep *P) {
  if (P->bwd_ready) return FAV_OK;
  for (PConv &pc : P->convs) {
    const int k = pc.k;
    std::vector<float> wt((size_t)pc.cin * pc.cout * k * k);
    for (int co = 0; co < pc.cout; ++co)
      for (int ci = 0; ci < pc.cin; ++ci)
        for (int ky = 0; ky < k; ++ky)
          for (int kx = 0; kx < k; ++kx)
            wt[(((size_t)ci * pc.cout + co) * k + ky) * k + kx] = pc.w[(((size_t)co * pc.cin + ci) * k + (k - 1 - ky)) * k + (k - 1 - kx)];
    std::vector<ConvDef> blocks;
    for (int b = 0; b < conv_nblocks(pc.cin); ++b) {
      ConvDef c;
      init_nblock_conv_def(c, "percep_dgrad" + std::to_string(pc.module), pc.cout, pc.cin, k, 1, pc.pad, b);
      if (build_phase_tables(c, c.phases[0]) != FAV_OK) {
        set_error("loss network module %d: the input gradient (convolution %d->%d k%d) is not a geometry the tensor-core planner runs",
                  pc.module, pc.cout, pc.cin, k);
        return FAV_ERR_UNSUPPORTED;
      }
      std::vector<uint16_t> pk = pack_phase_weights(c, c.phases[0], conv_nblock_weights(wt, pc.cout, pc.cin, k, b));
      void *d = nullptr;
      FAV_TRY(p_alloc(P->allocs, &d, pk.size() * 2));
      FAV_TRY(check_cuda(cudaMemcpy(d, pk.data(), pk.size() * 2, cudaMemcpyHostToDevice), "cudaMemcpy(percep dgrad weights)"));
      c.phases[0].d_b_tc = reinterpret_cast<uint4 *>(d);
      blocks.push_back(std::move(c));
    }
    if (!pc.d_zero) FAV_TRY(p_alloc(P->allocs, (void **)&pc.d_zero, kMaxNBlock * sizeof(float)));
    pc.dblocks = std::move(blocks);
  }
  P->bwd_ready = true;
  return FAV_OK;
}

// PerceptualCriterion:updateGradInput (PerceptualCriterion.lua:158-161): the loss layers' gradients, then from the deepest
// convolution back to the input.  Stage s: gradient at conv s's raw output (percep_bwd_stage_kernel), x 2^k into the operand of its
// input-gradient convolution, which writes the (scaled) gradient at conv s's input for stage s - 1 or grad_input.
static int run_backward(fav_percep *P, PPlan &pl, float *grad_input, cudaStream_t st) {
  const int ns = (int)P->convs.size();
  std::vector<int> written(P->taps.size(), 0);
  for (size_t k = 0; k < P->content_tap.size(); ++k) {
    const int t = P->content_tap[k];
    const PTap &a = pl.taps[1][t], &b = pl.taps[0][t];
    const int64_t HW = (int64_t)a.H * a.W;
    const float coef = (float)(P->content_w[k] * 2.0 / ((double)a.C * HW));
    percep_content_grad_kernel<<<dim3((unsigned)ceil_div64(HW, 256), a.C), 256, 0, st>>>(
        reinterpret_cast<const uint16_t *>(a.hi), reinterpret_cast<const uint16_t *>(a.lo), reinterpret_cast<const uint16_t *>(b.hi),
        reinterpret_cast<const uint16_t *>(b.lo), a.Cp, HW, coef, written[t], pl.tgrad[t]);
    FAV_TRY(post_launch("percep_content_grad"));
    written[t] = 1;
  }
  for (size_t k = 0; k < P->style_tap.size(); ++k) {
    const int t = P->style_tap[k];
    const PTap &a = pl.taps[1][t];
    const int64_t HW = (int64_t)a.H * a.W;
    if (P->agg == 1) {
      percep_mean_grad_kernel<<<dim3((unsigned)ceil_div64(HW, 256), a.C), 256, 0, st>>>(
          P->stat[k], P->target[k], HW, P->style_w[k] * 2.0 / ((double)a.C * HW), written[t], pl.tgrad[t]);
      FAV_TRY(post_launch("percep_mean_grad"));
    } else {
      const double C = a.C;
      percep_gram_diff_kernel<<<ceil_div(a.C * a.C, 256), 256, 0, st>>>(P->stat[k], P->target[k], a.C * a.C,
                                                                        P->style_w[k] * 4.0 / (C * C * C * (double)HW), pl.gram_d);
      FAV_TRY(post_launch("percep_gram_diff"));
      percep_gram_grad_kernel<<<dim3((unsigned)ceil_div64(HW, kGbN), ceil_div(a.C, kGbM)), 256, 0, st>>>(
          pl.gram_d, a.hi, a.lo, a.C, a.Cp, HW, written[t], pl.tgrad[t]);
      FAV_TRY(post_launch("percep_gram_grad"));
    }
    written[t] = 1;
  }
  FAV_TRY(check_cuda(cudaMemsetAsync(pl.gmax, 0, (size_t)ns * sizeof(unsigned), st), "cudaMemsetAsync(gmax)"));
  for (int s = ns - 1; s >= 0; --s) {
    const RawTensor &r = pl.raw[s];
    BwdStage bs;
    memset(&bs, 0, sizeof(bs));
    bs.raw = reinterpret_cast<const float4 *>(r.p); bs.C = r.C; bs.Cq = r.Cq; bs.Wp = r.Wp; bs.H = r.H; bs.W = r.W;
    if (s + 1 < ns) {
      const PStageSpec &nx = P->next[s];
      const RawTensor &d = pl.gin[s + 1];
      bs.nxt = reinterpret_cast<const float4 *>(d.p); bs.nxt_Wp = d.Wp; bs.nxt_max = pl.gmax + s + 1;
      bs.t[bs.nt++] = BwdTerm{nullptr, d.H, d.W, nx.relu, nx.pool.on};
      if (nx.pool.on) bs.pool = nx.pool;
    }
    for (size_t t = 0; t < P->taps.size(); ++t) {
      const PTapSpec &ts = P->taps[t];
      if (ts.stage != s) continue;
      const PTap &tp = pl.taps[1][t];
      bs.t[bs.nt++] = BwdTerm{pl.tgrad[t], tp.H, tp.W, ts.relu, ts.pool.on};
      if (ts.pool.on) bs.pool = ts.pool;
    }
    bs.out = reinterpret_cast<float4 *>(pl.gbuf); bs.out_max = pl.gmax + s;
    percep_bwd_stage_kernel<<<dim3(ceil_div(r.W, 128), r.H, r.Cq), 128, 0, st>>>(bs);
    FAV_TRY(post_launch("percep_bwd_stage"));
    const Operand &o = pl.gop[s];
    percep_bwd_pack_kernel<<<dim3(ceil_div(o.W, 128), o.H, o.Cb), 128, 0, st>>>(reinterpret_cast<const float4 *>(pl.gbuf), r.Cq, r.Wp,
                                                                                pl.gmax + s, o);
    FAV_TRY(post_launch("percep_bwd_pack"));
    for (const ConvJob &j : pl.djobs[s]) FAV_TRY(launch_conv_tc(j, P->num_sms, st));
  }
  const RawTensor &d = pl.gin[0];
  percep_grad_input_kernel<<<(unsigned)ceil_div64((int64_t)pl.H * pl.W, 256), 256, 0, st>>>(
      reinterpret_cast<const float4 *>(d.p), d.Wp, pl.gmax, pl.H, pl.W, grad_input);
  return post_launch("percep_grad_input");
}

}  // namespace fav

// =====================================================================================================================
extern "C" {

int fav_percep_create(int n_modules, const int *modules8, int n_content, const int *content_layers, const double *content_weights,
                      int n_style, const int *style_layers, const double *style_weights, int agg_type, fav_percep_t **out) {
  FAV_REQUIRE(out && modules8 && n_modules > 0, "fav_percep_create: null argument");
  FAV_REQUIRE(n_content >= 0 && n_style >= 0 && n_content + n_style > 0, "fav_percep_create: no loss layers");
  FAV_REQUIRE((!n_content || (content_layers && content_weights)) && (!n_style || (style_layers && style_weights)),
              "fav_percep_create: null layer list");
  FAV_REQUIRE(agg_type == 0 || agg_type == 1, "fav_percep_create: agg_type must be 0 (gram) or 1 (mean)");
  std::unique_ptr<fav_percep> P(new fav_percep());
  P->agg = agg_type;
  int last = 0;
  for (int i = 0; i < n_content; ++i) last = std::max(last, content_layers[i]);
  for (int i = 0; i < n_style; ++i) last = std::max(last, style_layers[i]);
  for (int i = 0; i < n_content; ++i) FAV_REQUIRE(content_layers[i] >= 1, "fav_percep_create: layer index %d", content_layers[i]);
  for (int i = 0; i < n_style; ++i) FAV_REQUIRE(style_layers[i] >= 1, "fav_percep_create: layer index %d", style_layers[i]);
  FAV_REQUIRE(last <= n_modules, "fav_percep_create: layer %d, but the loss network has %d modules", last, n_modules);
  // trim_network (layer_utils.lua:146-165): nothing after the deepest loss layer runs
  for (int i = 0; i < last; ++i) {
    const int *m = modules8 + 8 * i;
    PModule pm;
    pm.kind = m[0];
    if (pm.kind == 0) {
      pm.cin = m[1]; pm.cout = m[2]; pm.k = m[3]; pm.stride = m[4]; pm.pad = m[5];
      if (pm.cin < 1 || pm.cout < 1 || pm.k < 1 || pm.k % 2 == 0 || pm.pad < 0 || pm.pad > pm.k / 2 ||
          !(pm.stride == 1 || (pm.stride == 2 && pm.k == 3 && pm.pad == 1)) || !(pm.cin <= 8 || pm.cin % 16 == 0)) {
        set_error("loss network module %d: convolution %d->%d k%d stride %d pad %d is not a geometry the tensor-core planner runs",
                  i + 1, pm.cin, pm.cout, pm.k, pm.stride, pm.pad);
        return FAV_ERR_UNSUPPORTED;
      }
    } else if (pm.kind == 2) {
      pm.pool = PoolSpec{1, m[1], m[2], m[3], m[4], m[5], m[6]};
      pm.ceil_mode = m[7];
      if (m[1] < 1 || m[2] < 1 || m[3] < 1 || m[4] < 1 || m[5] < 0 || m[6] < 0 || 2 * m[5] > m[1] || 2 * m[6] > m[2]) {
        set_error("loss network module %d: bad max-pooling geometry", i + 1);
        return FAV_ERR_INVALID;
      }
    } else if (pm.kind != 1) {
      set_error("loss network module %d: unsupported module kind %d", i + 1, pm.kind);
      return FAV_ERR_UNSUPPORTED;
    }
    P->mods.push_back(pm);
  }
  // stages: conv s, then ReLUs and at most one max-pooling before conv s + 1
  std::map<int, int> tap_of;  // module index -> tap slot
  {
    std::vector<int> idx;
    for (int i = 0; i < n_content; ++i) idx.push_back(content_layers[i]);
    for (int i = 0; i < n_style; ++i) idx.push_back(style_layers[i]);
    std::sort(idx.begin(), idx.end());
    idx.erase(std::unique(idx.begin(), idx.end()), idx.end());
    for (int v : idx) tap_of[v] = -1;
  }
  int prev_ch = 3;
  int relu = 0, pooled = 0, ceil_mode = 0;
  PoolSpec pool{0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < last; ++i) {
    const PModule &m = P->mods[i];
    if (m.kind == 0) {
      if (P->convs.empty() && m.cin != 3) {
        set_error("loss network module %d: the first convolution must take the 3 image channels (has %d)", i + 1, m.cin);
        return FAV_ERR_UNSUPPORTED;
      }
      if (m.cin != prev_ch) {
        set_error("loss network module %d: convolution takes %d channels, the previous layer gives %d", i + 1, m.cin, prev_ch);
        return FAV_ERR_INVALID;
      }
      if (!P->convs.empty()) P->next.push_back(PStageSpec{relu, pool, ceil_mode});
      PConv pc;
      pc.module = i + 1; pc.cin = m.cin; pc.cout = m.cout; pc.k = m.k; pc.stride = m.stride; pc.pad = m.pad;
      for (int b = 0; b < conv_nblocks(m.cout); ++b) {
        ConvDef c;
        init_nblock_conv_def(c, "percep" + std::to_string(i + 1), m.cin, m.cout, m.k, m.stride, m.pad, b);
        if (build_phase_tables(c, c.phases[0]) != FAV_OK) {
          set_error("loss network module %d: convolution %d->%d k%d stride %d pad %d is not a geometry the tensor-core planner runs",
                    i + 1, m.cin, m.cout, m.k, m.stride, m.pad);
          return FAV_ERR_UNSUPPORTED;
        }
        pc.blocks.push_back(std::move(c));
      }
      P->convs.push_back(std::move(pc));
      prev_ch = m.cout;
      relu = 0; pooled = 0; ceil_mode = 0; pool = PoolSpec{0, 0, 0, 0, 0, 0, 0};
    } else {
      if (P->convs.empty()) {
        set_error("loss network module %d: a %s before the first convolution is not supported", i + 1, m.kind == 1 ? "ReLU" : "max-pooling");
        return FAV_ERR_UNSUPPORTED;
      }
      if (m.kind == 1) relu = 1;
      else {
        if (pooled) {
          set_error("loss network module %d: two max-poolings without a convolution between them are not supported", i + 1);
          return FAV_ERR_UNSUPPORTED;
        }
        pooled = 1; pool = m.pool; ceil_mode = m.ceil_mode;
      }
    }
    auto t = tap_of.find(i + 1);
    if (t != tap_of.end()) {
      PTapSpec ts;
      ts.index = i + 1; ts.stage = (int)P->convs.size() - 1; ts.relu = relu; ts.pool = pool; ts.ceil_mode = ceil_mode;
      t->second = (int)P->taps.size();
      P->taps.push_back(ts);
    }
  }
  for (int i = 0; i < n_content; ++i) {
    const int slot = tap_of[content_layers[i]];
    P->taps[slot].content = true;
    P->content_tap.push_back(slot);
    P->content_w.push_back(content_weights[i]);
    P->last_content_stage = std::max(P->last_content_stage, P->taps[slot].stage);
  }
  for (int i = 0; i < n_style; ++i) {
    P->style_tap.push_back(tap_of[style_layers[i]]);
    P->style_w.push_back(style_weights[i]);
  }
  *out = P.release();
  return FAV_OK;
}

void fav_percep_destroy(fav_percep_t *p) { delete p; }

int fav_percep_set_conv(fav_percep_t *p, int module_index, const float *weight, int64_t weight_numel, const float *bias,
                        int64_t bias_numel) {
  FAV_REQUIRE(p && weight && bias, "fav_percep_set_conv: null argument");
  FAV_REQUIRE(!p->finalized, "fav_percep_set_conv: already finalized");
  for (PConv &c : p->convs)
    if (c.module == module_index) {
      FAV_REQUIRE(weight_numel == (int64_t)c.cout * c.cin * c.k * c.k && bias_numel == c.cout,
                  "fav_percep_set_conv: module %d expects %lld weights and %d biases", module_index,
                  (long long)c.cout * c.cin * c.k * c.k, c.cout);
      c.w.assign(weight, weight + weight_numel);
      c.b.assign(bias, bias + bias_numel);
      c.set = true;
      return FAV_OK;
    }
  set_error("fav_percep_set_conv: module %d is not a convolution of the trimmed loss network", module_index);
  return FAV_ERR_INVALID;
}

int fav_percep_finalize(fav_percep_t *p) {
  FAV_REQUIRE(p, "fav_percep_finalize: null argument");
  if (p->finalized) return FAV_OK;
  for (PConv &c : p->convs) FAV_REQUIRE(c.set, "fav_percep_finalize: convolution module %d has no weights", c.module);
  FAV_TRY(require_device());
  int dev = 0;
  cudaDeviceProp prop;
  FAV_TRY(check_cuda(cudaGetDevice(&dev), "cudaGetDevice"));
  FAV_TRY(check_cuda(cudaGetDeviceProperties(&prop, dev), "cudaGetDeviceProperties"));
  if (prop.major != 9) {
    set_error("libfav_b200 targets sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
    return FAV_ERR_UNSUPPORTED;
  }
  p->num_sms = prop.multiProcessorCount;
  for (PConv &pc : p->convs)
    for (size_t b = 0; b < pc.blocks.size(); ++b) {
      ConvDef &c = pc.blocks[b];
      const std::vector<float> w = conv_nblock_weights(pc.w, pc.cin, pc.cout, pc.k, (int)b);
      std::vector<uint16_t> pk = pack_phase_weights(c, c.phases[0], w);
      void *d = nullptr;
      FAV_TRY(p_alloc(p->allocs, &d, pk.size() * 2));
      FAV_TRY(check_cuda(cudaMemcpy(d, pk.data(), pk.size() * 2, cudaMemcpyHostToDevice), "cudaMemcpy(percep weights)"));
      c.phases[0].d_b_tc = reinterpret_cast<uint4 *>(d);
      std::vector<float> bias(c.Npad, 0.f);
      for (int i = 0; i < c.cout; ++i) bias[i] = pc.b[(size_t)b * kMaxNBlock + i];
      float *db = nullptr;
      FAV_TRY(p_alloc(p->allocs, (void **)&db, bias.size() * 4));
      FAV_TRY(check_cuda(cudaMemcpy(db, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy(percep bias)"));
      pc.d_bias.push_back(db);
    }
  for (size_t k = 0; k < p->style_tap.size(); ++k) {
    const int C = p->convs[p->taps[p->style_tap[k]].stage].cout;
    double *t = nullptr, *s = nullptr;
    FAV_TRY(p_alloc(p->allocs, (void **)&t, (size_t)agg_len(p, C) * sizeof(double)));
    FAV_TRY(p_alloc(p->allocs, (void **)&s, (size_t)agg_len(p, C) * sizeof(double)));
    p->target.push_back(t);
    p->stat.push_back(s);
  }
  FAV_TRY(p_alloc(p->allocs, (void **)&p->d_losses, (p->content_tap.size() + p->style_tap.size() + 1) * sizeof(double)));
  p->finalized = true;
  return FAV_OK;
}

int fav_percep_set_style_target(fav_percep_t *p, const float *rgb, int H, int W, void *stream) {
  FAV_REQUIRE(p && rgb, "fav_percep_set_style_target: null argument");
  FAV_REQUIRE(p->finalized, "fav_percep_set_style_target: call fav_percep_finalize first");
  cudaStream_t st = (cudaStream_t)stream;
  PPlan *pl;
  FAV_TRY(build_pplan(p, H, W, &pl));
  p->last_plan = pl;
  p->last_backward = false;
  FAV_TRY(check_cuda(cudaMemsetAsync(pl->overflow, 0, sizeof(int), st), "cudaMemsetAsync(overflow)"));
  FAV_TRY(run_pass(p, *pl, rgb, 1, st));
  for (size_t k = 0; k < p->style_tap.size(); ++k) FAV_TRY(aggregate(p, *pl, pl->taps[1][p->style_tap[k]], p->target[k], st));
  FAV_TRY(check_overflow(*pl, st));
  p->has_target = true;
  return FAV_OK;
}

int fav_percep_evaluate(fav_percep_t *p, const float *content, const float *stylized, int H, int W, double *content_loss,
                        double *style_loss, void *stream) {
  FAV_REQUIRE(p && content && stylized && content_loss && style_loss, "fav_percep_evaluate: null argument");
  FAV_REQUIRE(p->finalized, "fav_percep_evaluate: call fav_percep_finalize first");
  FAV_REQUIRE(p->has_target || p->style_tap.empty(), "fav_percep_evaluate: set the style target first");
  cudaStream_t st = (cudaStream_t)stream;
  PPlan *pl;
  FAV_TRY(build_pplan(p, H, W, &pl));
  p->last_plan = pl;
  p->last_backward = false;
  FAV_TRY(check_cuda(cudaMemsetAsync(pl->overflow, 0, sizeof(int), st), "cudaMemsetAsync(overflow)"));
  // PerceptualCriterion.lua:85-93 then :117-155: capture the content targets, then the evaluated image in loss mode
  if (!p->content_tap.empty()) FAV_TRY(run_pass(p, *pl, content, 0, st));
  FAV_TRY(run_pass(p, *pl, stylized, 1, st));
  FAV_TRY(launch_losses(p, *pl, st));
  return finish_losses(p, *pl, st, content_loss, style_loss, nullptr);
}

int fav_percep_forward_backward(fav_percep_t *p, const float *content_pre, const float *input_pre, int H, int W, float *grad_input,
                                double *content_loss, double *style_loss, double *layer_losses, void *stream) {
  FAV_REQUIRE(p && input_pre && grad_input && content_loss && style_loss, "fav_percep_forward_backward: null argument");
  FAV_REQUIRE(content_pre || p->content_tap.empty(), "fav_percep_forward_backward: the content layers need a content target");
  FAV_REQUIRE(p->finalized, "fav_percep_forward_backward: call fav_percep_finalize first");
  FAV_REQUIRE(p->has_target || p->style_tap.empty(), "fav_percep_forward_backward: set the style target first");
  if (const int m = bwd_unsupported_module(p)) {
    const PConv *pc = nullptr;
    for (const PConv &c : p->convs)
      if (c.module == m) pc = &c;
    set_error("loss network module %d: convolution k%d stride %d pad %d: the backward pass runs stride-1 convolutions with pad "
              "(k-1)/2 only", m, pc->k, pc->stride, pc->pad);
    return FAV_ERR_UNSUPPORTED;
  }
  if (const int m = bwd_crowded_stage(p)) {
    set_error("loss network module %d: too many loss layers between this convolution and the next (the backward pass takes %d, "
              "or %d after the deepest convolution)", m, kMaxStageTerms - 1, kMaxStageTerms);
    return FAV_ERR_UNSUPPORTED;
  }
  FAV_TRY(prepare_backward(p));
  cudaStream_t st = (cudaStream_t)stream;
  PPlan *pl;
  FAV_TRY(build_pplan(p, H, W, &pl, true));
  p->last_plan = pl;
  p->last_backward = true;
  FAV_TRY(check_cuda(cudaMemsetAsync(pl->overflow, 0, sizeof(int), st), "cudaMemsetAsync(overflow)"));
  // PerceptualCriterion.lua:117-134 (setContentTarget, then the input in loss mode), then :158-161
  if (!p->content_tap.empty()) FAV_TRY(run_pass(p, *pl, content_pre, 0, st, true));
  FAV_TRY(run_pass(p, *pl, input_pre, 1, st, true));
  FAV_TRY(launch_losses(p, *pl, st));
  FAV_TRY(run_backward(p, *pl, grad_input, st));
  return finish_losses(p, *pl, st, content_loss, style_loss, layer_losses);
}

int fav_pixel_loss_grad(const float *out2, const float *prev_warped_masked, const float *cert, int N, int H, int W, int type,
                        float weight, float *grad_accum, double *loss, void *stream) {
  FAV_REQUIRE(out2 && prev_warped_masked && cert && grad_accum && loss, "fav_pixel_loss_grad: null argument");
  FAV_REQUIRE(N >= 1 && H >= 1 && W >= 1, "fav_pixel_loss_grad: bad size %dx%dx%d", N, H, W);
  FAV_REQUIRE(type >= 0 && type <= 2, "fav_pixel_loss_grad: type must be 0 (L2), 1 (L1) or 2 (SmoothL1)");
  FAV_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t HW = (int64_t)H * W, n = 3 * (int64_t)N * HW;
  // the criterion's norm (THNN MSECriterion 2/n, AbsCriterion and SmoothL1Criterion 1/n), in fp32 as its `real`
  const float norm = (float)((type == 0 ? 2.0 : 1.0) / (double)n);
  double *part = nullptr;
  FAV_TRY(check_cuda(cudaMallocAsync((void **)&part, (kRedBlocks + 1) * sizeof(double), st), "cudaMallocAsync(pixel loss)"));
  fav_pixel_loss_grad_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(out2, prev_warped_masked, cert, HW, n, type, norm, weight, grad_accum, part);
  int rc = post_launch("fav_pixel_loss_grad");
  if (rc == FAV_OK) {
    percep_sum_kernel<<<1, kRedThreads, 0, st>>>(part, kRedBlocks, (double)weight / (double)n, part + kRedBlocks);
    rc = post_launch("percep_sum");
  }
  if (rc == FAV_OK)
    rc = check_cuda(cudaMemcpyAsync(loss, part + kRedBlocks, sizeof(double), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync(pixel loss)");
  const int rf = check_cuda(cudaFreeAsync(part, st), "cudaFreeAsync(pixel loss)");
  if (rc == FAV_OK) rc = rf;
  if (rc == FAV_OK) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize(pixel loss)");
  return rc;
}

int fav_tv_grad(const float *x, int N, int H, int W, float strength, float *grad_accum, void *stream) {
  FAV_REQUIRE(x && grad_accum, "fav_tv_grad: null argument");
  FAV_REQUIRE(N >= 1 && H >= 1 && W >= 1, "fav_tv_grad: bad size %dx%dx%d", N, H, W);
  FAV_TRY(require_device());
  const int64_t planes = 3 * (int64_t)N, total = planes * H * W;
  fav_tv_grad_kernel<<<(unsigned)ceil_div64(total, 256), 256, 0, (cudaStream_t)stream>>>(x, planes, H, W, strength, grad_accum);
  return post_launch("fav_tv_grad");
}

int fav_percep_layer_output(fav_percep_t *p, int pass, int index, float *out, int *C, int *Hl, int *Wl, void *stream) {
  FAV_REQUIRE(p && p->last_plan, "fav_percep_layer_output: run an evaluation or set a style target first");
  FAV_REQUIRE(pass == 0 || pass == 1, "fav_percep_layer_output: pass must be 0 (content target) or 1 (evaluated image)");
  PPlan *pl = p->last_plan;
  for (size_t t = 0; t < p->taps.size(); ++t)
    if (p->taps[t].index == index) {
      const PTap &tp = pl->taps[pass][t];
      FAV_REQUIRE(tp.hi, "fav_percep_layer_output: layer %d is not a content layer (pass 0 keeps those only)", index);
      if (C) *C = tp.C;
      if (Hl) *Hl = tp.H;
      if (Wl) *Wl = tp.W;
      if (!out) return FAV_OK;
      const int64_t P = (int64_t)tp.H * tp.W;
      percep_unpack_tap_kernel<<<dim3((unsigned)ceil_div64(P, 256), tp.C), 256, 0, (cudaStream_t)stream>>>(
          reinterpret_cast<const uint16_t *>(tp.hi), reinterpret_cast<const uint16_t *>(tp.lo), tp.Cp, tp.C, P, out);
      return post_launch("percep_unpack_tap");
    }
  set_error("fav_percep_layer_output: layer %d is not a loss layer", index);
  return FAV_ERR_INVALID;
}

int fav_percep_conv_output(fav_percep_t *p, int module_index, float *out, int *C, int *H, int *W, void *stream) {
  FAV_REQUIRE(p && p->last_plan && p->last_backward, "fav_percep_conv_output: the last call was not fav_percep_forward_backward");
  const PPlan *pl = p->last_plan;
  for (size_t s = 0; s < p->convs.size(); ++s)
    if (p->convs[s].module == module_index) {
      const RawTensor &r = pl->raw[s];
      if (C) *C = r.C;
      if (H) *H = r.H;
      if (W) *W = r.W;
      if (!out) return FAV_OK;
      percep_unpack_raw_kernel<<<dim3((unsigned)ceil_div64((int64_t)r.H * r.W, 256), r.C), 256, 0, (cudaStream_t)stream>>>(
          r.p, r.Cq, r.Wp, r.C, r.H, r.W, out);
      return post_launch("percep_unpack_raw");
    }
  set_error("fav_percep_conv_output: module %d is not a convolution of the trimmed loss network", module_index);
  return FAV_ERR_INVALID;
}

int fav_percep_style_stat(fav_percep_t *p, int which, int k, double *out, int *n, void *stream) {
  FAV_REQUIRE(p && p->finalized, "fav_percep_style_stat: finalize first");
  FAV_REQUIRE(which == 0 || which == 1, "fav_percep_style_stat: which must be 0 (style target) or 1 (last evaluated image)");
  FAV_REQUIRE(k >= 0 && k < (int)p->style_tap.size(), "fav_percep_style_stat: style layer %d out of range", k);
  const int len = agg_len(p, p->convs[p->taps[p->style_tap[k]].stage].cout);
  if (n) *n = len;
  if (!out) return FAV_OK;
  return check_cuda(cudaMemcpyAsync(out, (which == 0 ? p->target : p->stat)[k], (size_t)len * sizeof(double),
                                    cudaMemcpyDeviceToDevice, (cudaStream_t)stream),
                    "cudaMemcpyAsync(style stat)");
}
}
