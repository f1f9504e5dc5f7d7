// net_layout.cuh -- HBM data layouts of the stylization net (fast_artistic_video/models_video.lua:55-140).
//
// The reference keeps every activation as fp32 NCHW.  Internally this implementation uses two layouts,
// both chosen so that the wgmma implicit-GEMM convolution needs neither im2col nor swizzled TMA maps:
//
//  Operand  activation feeding a convolution, stored as an fp16 PAIR (hi, lo) with x ~= hi + lo
//           (22 significant bits).  Layout per tensor: [Hs][Cb][Ws][8 channels] -- 16 bytes per
//           (pixel, channel-block).  A run of consecutive pixels of one channel block is contiguous in
//           HBM *and* is exactly the canonical no-swizzle K-major UMMA core-matrix layout (8 rows x 16 B),
//           so a 1-D bulk copy (cp.async.bulk) of a row segment lands MMA-ready in shared memory and a
//           filter tap is just a +16 B * dx offset of the matrix descriptor's start address.
//           Zero padding of the convolution is materialised as a zero border (padT/padL + slack).
//           Inputs of stride-2 convolutions are stored parity-split: [Hs][Cb][2][Ws2][8]
//           (even x plane, then odd x plane) so that stride-2 taps stay contiguous.
//  Raw      fp32 convolution output before InstanceNorm: [Ho][Cq][Wp][4 channels] -- 16 bytes per
//           (pixel, channel-quad); the epilogue writes the two channels a thread holds as one 8-byte store.
//           RawTensor::planar (fp32 [C][Hp][Wp]) is a layout the normalisation kernels also accept.
#pragma once
#include "fav_common.cuh"
#include <cuda_fp16.h>

namespace fav {

struct Operand {
  __half *hi = nullptr, *lo = nullptr;
  int C = 0, Cb = 0;        // logical channels, channel blocks of 8 (zero padded)
  int H = 0, W = 0;         // logical size
  int padT = 0, padL = 0;   // storage coords of logical (0,0)
  int Hs = 0, Ws = 0;       // storage rows / pixels per (row, cb) slab (non-parity)
  int parity = 0, Ws2 = 0;  // parity split: slab = [2][Ws2]
  size_t elems16 = 0;       // allocation size in 16-byte units (per hi / lo), incl. tail slack
  __host__ __device__ int slab16() const { return parity ? 2 * Ws2 : Ws; }
  // offset in 16-byte units of storage pixel (ys, xs) of channel block cb
  __host__ __device__ int64_t off16(int ys, int cb, int xs) const {
    int64_t base = ((int64_t)ys * Cb + cb) * slab16();
    return base + (parity ? (int64_t)(xs & 1) * Ws2 + (xs >> 1) : xs);
  }
};

#ifdef __CUDACC__
// 8 fp32 channels of one pixel -> fp16 hi / lo halves (x ~= hi + lo), 16 bytes each
// x ~= hi + lo with both halves fp16: two packed conversions per channel pair (F2FP.SATFINITE.F16.F32.PACK_AB, HADD2.F32 x2,
// FADD x2, F2FP) -- 3 instructions per value.  satfinite replaces the explicit clamp to +-65504 (same values for every
// finite |x| <= 65504; InstanceNorm outputs are bounded by gamma * sqrt(H*W)).  a -> low 16 bits, b -> high 16 bits.
__device__ __forceinline__ void split_pair(float a, float b, uint32_t &h, uint32_t &l) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2 *>(&h));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(l) : "f"(b - hf.y), "f"(a - hf.x));
}

__device__ __forceinline__ void split_store8(const float v[8], uint4 *hi_dst, uint4 *lo_dst) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_pair(v[2 * i], v[2 * i + 1], h[i], l[i]);
  *hi_dst = make_uint4(h[0], h[1], h[2], h[3]);
  *lo_dst = make_uint4(l[0], l[1], l[2], l[3]);
}

// gamma / sqrt(var + eps) of InstanceNormalization.lua:39-50 (biased variance, eps inside the root), from the double sums
// of the fused statistics: ONE definition for in_apply, up_apply and the norm-on-load tables of both conv kernels.
// rsqrt + multiply instead of sqrt + divide: about half the dependent double-precision instruction chain that every block
// waits for; the result is rounded to float afterwards.
__device__ __forceinline__ void in_finalize(double sum, double sumsq, double inv_count, double eps, float gamma, float &mean_f,
                                            float &scale_f) {
  const double mean = sum * inv_count;
  double var = sumsq * inv_count - mean * mean;
  if (var < 0) var = 0;
  mean_f = (float)mean;
  scale_f = (float)((double)gamma * rsqrt(var + eps));
}

#endif

struct RawTensor {
  float *p = nullptr;
  int C = 0, Cq = 0;  // channels, channel quads
  int H = 0, W = 0;   // logical size
  int Hp = 0, Wp = 0; // allocated rows / row pitch in pixels (multiple of 128; planar: multiple of 16)
  int planar = 0;     // 1: fp32 [C][Hp][Wp]; 0: [Ho][Cq][Wp][4]
  __host__ __device__ int64_t off4(int y, int cq, int x) const { return (((int64_t)y * Cq + cq) * Wp + x); }
  __host__ __device__ int64_t offp(int c, int y, int x) const { return (((int64_t)c * Hp + y) * Wp + x); }
};

// one filter tap of a (phase of a) convolution: input pixel = (sy*y + dy, sx*x + dx)
struct ConvTap {
  int dy, dx;
  int ky, kx;  // index into the Torch weight tensor
};

}  // namespace fav
