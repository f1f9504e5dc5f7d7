// consistency.cu -- forward/backward-flow occlusion test on the GPU.
//   a-11 checkConsistency          consistencyChecker/consistencyChecker.cpp:80-134
//   a-12 computeCorners + normalize + avg    consistencyChecker.cpp:39-78, CMatrix.h:721-736,1245-1251,
//        filters CFilter.h:600-611 (taps), :1499-1578 (mirror borders), :1417-1464 (IIR)
//
// The reference evaluates hard thresholds with a mix of float and double arithmetic (:110-125).  The
// kernels below mirror that mix operation by operation with explicit round-to-nearest intrinsics (no
// FMA contraction), so the {0,255} mask is BIT-IDENTICAL to the reference binary's PGM.  The work is a
// 2-plane gather + one byte store per pixel: HBM-bound, 4 pixels per thread, 16-byte flow1 loads.
//
// The motion-edge branch (:129-132) assigns MOTION_BOUNDARIE_VALUE = 255 (:12) to pixels that are
// already 255 and is therefore not evaluated (no observable effect).
#include "fav_common.cuh"
#include "exact_avg.cuh"
#include "occlusion.cuh"

namespace fav {

__global__ void __launch_bounds__(256) consistency_kernel(const float *__restrict__ f1u, const float *__restrict__ f1v,
                                                          const float *__restrict__ f2u, const float *__restrict__ f2v,
                                                          const float *__restrict__ structure,
                                                          const float *__restrict__ avg_dev, float avg_host,
                                                          uint8_t *__restrict__ rel, float *__restrict__ cert, int W,
                                                          int H, int vec) {
  int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * vec;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x0 >= W || y >= H) return;
  const int64_t o = (int64_t)y * W + x0;
  float savg = avg_dev ? __ldg(avg_dev) : avg_host;
  float u2[4], v2[4];
  if (vec == 4) {
    float4 t = __ldg(reinterpret_cast<const float4 *>(f1u + o));
    u2[0] = t.x; u2[1] = t.y; u2[2] = t.z; u2[3] = t.w;
    t = __ldg(reinterpret_cast<const float4 *>(f1v + o));
    v2[0] = t.x; v2[1] = t.y; v2[2] = t.z; v2[3] = t.w;
  } else {
    u2[0] = f1u[o];
    v2[0] = f1v[o];
  }
  uint8_t r[4];
  for (int i = 0; i < vec; ++i)
    r[i] = check_pixel(f2u, f2v, u2[i], v2[i], x0 + i, y, W, H, structure, savg);
  if (vec == 4) {
    if (rel) *reinterpret_cast<uchar4 *>(rel + o) = make_uchar4(r[0], r[1], r[2], r[3]);
    if (cert)
      *reinterpret_cast<float4 *>(cert + o) =
          make_float4(r[0] ? 1.f : 0.f, r[1] ? 1.f : 0.f, r[2] ? 1.f : 0.f, r[3] ? 1.f : 0.f);
  } else {
    if (rel) rel[o] = r[0];
    if (cert) cert[o] = r[0] ? 1.f : 0.f;  // image.load(pgm,1): byte/255 (fast_artistic_video.lua:103)
  }
}

int launch_consistency(const float *f1u, const float *f1v, const float *f2u, const float *f2v, const float *structure,
                       const float *avg_dev, float avg_host, uint8_t *rel, float *cert, int W, int H, cudaStream_t st) {
  auto al = [](const void *p, int a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
  int vec = (W % 4 == 0 && al(f1u, 16) && al(f1v, 16) && (!rel || al(rel, 4)) && (!cert || al(cert, 16))) ? 4 : 1;
  dim3 block(32, 8), grid(ceil_div(ceil_div(W, vec), 32), ceil_div(H, 8));
  consistency_kernel<<<grid, block, 0, st>>>(f1u, f1v, f2u, f2v, structure, avg_dev, avg_host, rel, cert, W, H, vec);
  return post_launch("checkConsistency");
}

// ---------------------------------------------------------------------------------------------------
// a-12 computeCorners (4-argument mode).  Stages:
//   1. per-pixel structure tensor from 3-tap central differences with mirrored borders (fully parallel)
//   2. Deriche-style IIR along X (one thread per row) then along Y (one thread per column, coalesced)
//      for dxx, dyy, dxy -- the recurrences are sequential per line, as in the reference
//   3. smallest eigenvalue (parallel)
//   4. normalize(0,1): the reference's `else if` min/max scan is evaluated EXACTLY by a parallel prefix-maximum scan
//      (norm_*_kernel); the fp32 avg, order-dependent by rounding, EXACTLY by integer runs within a binade (exact_avg.cuh,
//      avg_*_kernel).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float deriv3(float m1, float c0, float p1) {
  // sum over i=-1,0,1 of f[i]*v starting from 0 (CFilter.h:1510-1514): ((0 + -0.5*m1) + 0*c0) + 0.5*p1
  float s = __fadd_rn(0.f, __fmul_rn(-0.5f, m1));
  s = __fadd_rn(s, __fmul_rn(0.0f, c0));
  s = __fadd_rn(s, __fmul_rn(0.5f, p1));
  return s;
}

// scale: the image planes times `scale` are CTensor's 0..255 planes (1 for such planes; 255 for a frame of byte/255 values,
// where fl(fl(byte/255) * 255) == byte for every byte)
__global__ void __launch_bounds__(256) structure_tensor_kernel(const float *__restrict__ img, float scale, int Z, int W, int H,
                                                               float *__restrict__ dxx, float *__restrict__ dyy,
                                                               float *__restrict__ dxy) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  int64_t n = (int64_t)W * H, o = (int64_t)y * W + x;
  // mirrored neighbours: x-1<0 -> -1-(x-1) = 0 ; x+1>=W -> 2W-1-(x+1) = W-1   (CFilter.h:1511-1512)
  int xm = x - 1 < 0 ? 0 : x - 1, xp = x + 1 >= W ? W - 1 : x + 1;
  int ym = y - 1 < 0 ? 0 : y - 1, yp = y + 1 >= H ? H - 1 : y + 1;
  float sxx = 0.f, syy = 0.f, sxy = 0.f;
  for (int k = 0; k < Z; ++k) {  // consistencyChecker.cpp:55-61
    const float *p = img + k * n;
    float c0 = __fmul_rn(__ldg(p + o), scale);
    float gx = deriv3(__fmul_rn(__ldg(p + (int64_t)y * W + xm), scale), c0, __fmul_rn(__ldg(p + (int64_t)y * W + xp), scale));
    float gy = deriv3(__fmul_rn(__ldg(p + (int64_t)ym * W + x), scale), c0, __fmul_rn(__ldg(p + (int64_t)yp * W + x), scale));
    sxx = __fadd_rn(sxx, __fmul_rn(gx, gx));
    syy = __fadd_rn(syy, __fmul_rn(gy, gy));
    sxy = __fadd_rn(sxy, __fmul_rn(gx, gy));
  }
  dxx[o] = sxx; dyy[o] = syy; dxy[o] = sxy;
}

struct IirC { float k, pm, pp, e2, te; };
constexpr int kIirChunk = 16;

// 32 x 32 tiled transpose of 3 planes (blockIdx.z): the X pass of the IIR runs on the transposed matrices so that the
// one-thread-per-line recurrence reads and writes coalesced (neighbouring threads = neighbouring lines = neighbouring addresses)
__global__ void __launch_bounds__(256) transpose3_kernel(const float *__restrict__ in, float *__restrict__ out, int rows, int cols,
                                                         int64_t plane) {
  __shared__ float tile[32][33];
  const float *src = in + blockIdx.z * plane;
  float *dst = out + blockIdx.z * plane;
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8)
    if (by + r < rows && bx + tx < cols) tile[r][tx] = src[(int64_t)(by + r) * cols + bx + tx];
  __syncthreads();
  for (int r = ty; r < 32; r += 8)
    if (bx + r < cols && by + tx < rows) dst[(int64_t)(bx + r) * rows + by + tx] = tile[tx][r];
}

// one thread per line; `stride` between consecutive samples of the line, `pitch` between lines.
// v1 scratch holds the causal pass (CFilter.h:1428-1431), the anti-causal pass (:1432-1435) is fused
// with the final sum (:1436-1437).  3 matrices per launch via blockIdx.y.
__global__ void __launch_bounds__(128) iir_kernel(float *__restrict__ m0, float *__restrict__ m1p,
                                                  float *__restrict__ m2p, float *__restrict__ scratch, int n,
                                                  int lines, int64_t stride, int64_t pitch, int64_t plane, IirC c) {
  int line = blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= lines) return;
  float *m = blockIdx.y == 0 ? m0 : (blockIdx.y == 1 ? m1p : m2p);
  float *src = m + line * pitch;
  float *v1 = scratch + blockIdx.y * plane + line * pitch;
#define S(i) src[(int64_t)(i) * stride]
#define V1(i) v1[(int64_t)(i) * stride]
  const float k = c.k, pm = c.pm, pp = c.pp, e2 = c.e2, te = c.te;
  float a0 = __fmul_rn(__fsub_rn(0.5f, __fmul_rn(k, pm)), S(0));
  V1(0) = a0;
  float s_prev = S(0), s_cur = S(1);
  float a1 = __fadd_rn(__fmul_rn(k, __fadd_rn(s_cur, __fmul_rn(pm, s_prev))), __fmul_rn(__fsub_rn(te, e2), a0));
  V1(1) = a1;
  // the recurrence is sequential per line, the memory accesses are not: kIirChunk samples are requested ahead of the chain
  for (int xb = 2; xb < n; xb += kIirChunk) {
    float sv[kIirChunk];
#pragma unroll
    for (int j = 0; j < kIirChunk; ++j) sv[j] = xb + j < n ? S(xb + j) : 0.f;
#pragma unroll
    for (int j = 0; j < kIirChunk; ++j) {
      if (xb + j >= n) break;
      s_prev = s_cur;
      s_cur = sv[j];
      float a = __fsub_rn(__fadd_rn(__fmul_rn(k, __fadd_rn(s_cur, __fmul_rn(pm, s_prev))), __fmul_rn(te, a1)),
                          __fmul_rn(e2, a0));
      V1(xb + j) = a;
      a0 = a1;
      a1 = a;
    }
  }
  // anti-causal
  float sN1 = S(n - 1);
  float b0 = __fmul_rn(__fadd_rn(0.5f, __fmul_rn(k, pm)), sN1);                        // v2[n-1]
  float b1 = __fadd_rn(__fmul_rn(k, __fmul_rn(__fsub_rn(pp, e2), sN1)), __fmul_rn(__fsub_rn(te, e2), b0));  // v2[n-2]
  float s_p1 = S(n - 2), s_p2 = sN1;  // S(x+1), S(x+2) for x = n-3
  S(n - 1) = __fadd_rn(V1(n - 1), b0);
  // S(n-2) is still needed as S(x+1) for x = n-3: it is cached in s_p1
  S(n - 2) = __fadd_rn(V1(n - 2), b1);
  for (int xb = n - 3; xb >= 0; xb -= kIirChunk) {
    float sv[kIirChunk], vv[kIirChunk];
#pragma unroll
    for (int j = 0; j < kIirChunk; ++j) { sv[j] = xb - j >= 0 ? S(xb - j) : 0.f; vv[j] = xb - j >= 0 ? V1(xb - j) : 0.f; }
#pragma unroll
    for (int j = 0; j < kIirChunk; ++j) {
      if (xb - j < 0) break;
      float b = __fsub_rn(__fadd_rn(__fmul_rn(k, __fsub_rn(__fmul_rn(pp, s_p1), __fmul_rn(e2, s_p2))), __fmul_rn(te, b1)),
                          __fmul_rn(e2, b0));
      S(xb - j) = __fadd_rn(vv[j], b);
      s_p2 = s_p1;
      s_p1 = sv[j];
      b0 = b1;
      b1 = b;
    }
  }
#undef S
#undef V1
}

__global__ void __launch_bounds__(256) eigen_kernel(const float *__restrict__ dxx, const float *__restrict__ dxy,
                                                    const float *__restrict__ dyy, float *__restrict__ corners,
                                                    int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = dxx[i], b = dxy[i], c = dyy[i];
  float temp = (float)__dmul_rn(0.5, (double)__fadd_rn(a, c));  // :73  0.5*(a+c)
  float temp2 = __fsub_rn(__fadd_rn(__fmul_rn(temp, temp), __fmul_rn(b, b)), __fmul_rn(a, c));
  // :75-76  temp - sqrt(temp2): double sqrt, difference formed in double, rounded once (pinned to _ref)
  corners[i] = (temp2 < 0.0f) ? 0.0f : (float)__dsub_rn((double)temp, __dsqrt_rn((double)temp2));
}

// CMatrix::normalize's scan (CMatrix.h:721-736):  if (v > max) max = v; else if (v < min) min = v;
// max is the plain maximum (floor -30000).  An element that raises the running maximum is NOT offered to the minimum, so
//   min = min(30000, { v_i : v_i <= max(-30000, v_0..v_{i-1}) }):
// the minimum over the elements that are not strict prefix maxima.  Prefix maximum is an associative scan, so the quirk
// parallelises exactly: per-block maxima -> exclusive prefix maximum over the blocks -> per-block rescan with the carry.
constexpr int kNormBlock = 1024;
__global__ void __launch_bounds__(kNormBlock) norm_block_max_kernel(const float *__restrict__ m, int64_t n, float *__restrict__ bmax) {
  const int64_t i = (int64_t)blockIdx.x * kNormBlock + threadIdx.x;
  float v = i < n ? m[i] : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __shared__ float red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (threadIdx.x == 0) bmax[blockIdx.x] = v;
  }
}
// one block: carry[b] = max(-30000, maxima of blocks < b) (exclusive), carry[nb] = the total
__global__ void __launch_bounds__(1024) norm_carry_kernel(const float *__restrict__ bmax, int nb, float *__restrict__ carry) {
  __shared__ float part[1024];
  const int per = (nb + 1023) / 1024, b0 = threadIdx.x * per;
  float loc = -INFINITY;
  for (int b = b0; b < min(nb, b0 + per); ++b) loc = fmaxf(loc, bmax[b]);
  part[threadIdx.x] = loc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float run = -30000.f;  // CMatrix.h:722 initial maximum
    for (int t = 0; t < 1024; ++t) { const float v = part[t]; part[t] = run; run = fmaxf(run, v); }
    carry[nb] = run;
  }
  __syncthreads();
  float run = part[threadIdx.x];
  for (int b = b0; b < min(nb, b0 + per); ++b) { carry[b] = run; run = fmaxf(run, bmax[b]); }
}
__global__ void __launch_bounds__(kNormBlock) norm_block_min_kernel(const float *__restrict__ m, int64_t n, const float *__restrict__ carry,
                                                                    float *__restrict__ bmin) {
  const int64_t i = (int64_t)blockIdx.x * kNormBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const float v = i < n ? m[i] : -INFINITY;
  // exclusive prefix maximum inside the block: warp scan, then the warps' totals
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc = fmaxf(inc, t); }
  float exc = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) exc = -INFINITY;
  __shared__ float wtot[32], red[32];
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  float before = carry[blockIdx.x];
  for (int k = 0; k < w; ++k) before = fmaxf(before, wtot[k]);
  const float pmax = fmaxf(before, exc);              // max(-30000, v_0 .. v_{i-1})
  float cand = (i < n && !(v > pmax)) ? v : INFINITY;  // the `else if (v < min)` branch sees v only when it did not raise max
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cand = fminf(cand, __shfl_xor_sync(0xffffffffu, cand, o));
  if (lane == 0) red[w] = cand;
  __syncthreads();
  if (threadIdx.x < 32) {
    cand = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cand = fminf(cand, __shfl_xor_sync(0xffffffffu, cand, o));
    if (threadIdx.x == 0) bmin[blockIdx.x] = cand;
  }
}
__global__ void __launch_bounds__(1024) norm_final_kernel(const float *__restrict__ bmin, int nb, const float *__restrict__ carry,
                                                          float *__restrict__ minmax) {
  float v = INFINITY;
  for (int b = threadIdx.x; b < nb; b += 1024) v = fminf(v, bmin[b]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __shared__ float red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float cmin = 30000.f;  // CMatrix.h:722 initial minimum
    for (int k = 0; k < 32; ++k) cmin = fminf(cmin, red[k]);
    const float cmax = carry[nb];
    float t = __fsub_rn(cmax, cmin);  // :729-731
    if (t == 0.f) t = 1.f;
    else t = __fdiv_rn(1.0f, t);
    minmax[0] = cmin;
    minmax[1] = t;
  }
}
__global__ void __launch_bounds__(256) normalize_apply_kernel(float *__restrict__ m, int64_t n,
                                                              const float *__restrict__ minmax) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = __fsub_rn(m[i], minmax[0]);
  v = __fmul_rn(v, minmax[1]);
  m[i] = __fadd_rn(v, 0.0f);
}
// CMatrix::avg (CMatrix.h:1245-1251) adds the elements IN ORDER in fp32: every partial sum is rounded, so the result depends on
// the order.  Evaluated exactly in parallel (exact_avg.cuh): double sums of the sub-chunks and chunks (the estimate that picks
// the hypotheses) -> one block per chunk runs every (sub-chunk, hypothesis) in integers and composes the chunk's records -> one
// warp combines the chunks in order from the exact state.
struct AvgWs {
  double *ssum, *csum;
  AvgRec *srec, *crec;
  int64_t nsub;
  int nch;
};
__host__ __device__ inline size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }
static size_t avg_ws_bytes(int64_t n) {
  const int64_t nsub = ceil_div64(n, kAvgSub), nch = ceil_div64(nsub, kAvgGroup);
  return align16(nsub * sizeof(double)) + align16(nch * sizeof(double)) + align16(nsub * sizeof(AvgRec)) +
         align16(nch * sizeof(AvgRec)) + 16;
}
static AvgWs avg_ws(void *base, int64_t n) {
  AvgWs w;
  w.nsub = ceil_div64(n, kAvgSub);
  w.nch = (int)ceil_div64(w.nsub, kAvgGroup);
  char *p = (char *)(((uintptr_t)base + 15) & ~(uintptr_t)15);
  w.ssum = (double *)p; p += align16(w.nsub * sizeof(double));
  w.csum = (double *)p; p += align16(w.nch * sizeof(double));
  w.srec = (AvgRec *)p; p += align16(w.nsub * sizeof(AvgRec));
  w.crec = (AvgRec *)p;
  return w;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one block per chunk: the double sum of each sub-chunk and of the chunk
__global__ void __launch_bounds__(256) avg_sum_kernel(const float *__restrict__ m, int64_t n, double *__restrict__ ssum,
                                                      double *__restrict__ csum) {
  __shared__ double part[8];
  const int c = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t nsub = ceil_div64(n, kAvgSub);
  double cs = 0.0;
  for (int g = w; g < kAvgGroup; g += 8) {
    const int64_t s = (int64_t)c * kAvgGroup + g;
    if (s >= nsub) break;
    double v = 0.0;
    for (int i = lane; i < kAvgSub; i += 32) {
      const int64_t e = s * kAvgSub + i;
      if (e < n) v += (double)__ldg(m + e);
    }
    v = warp_sum_d(v);
    if (lane == 0) ssum[s] = v;
    cs += v;
  }
  if (lane == 0) part[w] = cs;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += part[k];
    csum[c] = t;
  }
}

// one block per chunk, one thread per (sub-chunk, hypothesis): the sub-chunks' records, then the chunk's records composed from them
constexpr int kAvgHypThreads = kAvgGroup * kAvgHyps;
__global__ void __launch_bounds__(kAvgHypThreads) avg_hyp_kernel(const float *__restrict__ m, int64_t n,
                                                                 const double *__restrict__ ssum, const double *__restrict__ csum,
                                                                 AvgRec *__restrict__ srec, AvgRec *__restrict__ crec) {
  __shared__ double red[kAvgHypThreads / 32];
  __shared__ int32_t seb[kAvgGroup];
  __shared__ AvgHyp sh[kAvgGroup][kAvgHyps];
  const int c = blockIdx.x, t = threadIdx.x;
  const int64_t nsub = ceil_div64(n, kAvgSub), s0 = (int64_t)c * kAvgGroup;
  const int ns = (int)min((int64_t)kAvgGroup, nsub - s0);
  double p = 0.0;  // the estimate of the running sum before this chunk
  for (int i = t; i < c; i += kAvgHypThreads) p += csum[i];
  p = warp_sum_d(p);
  if ((t & 31) == 0) red[t >> 5] = p;
  __syncthreads();
  if (t == 0) {
    double S = 0.0;
    for (int k = 0; k < kAvgHypThreads / 32; ++k) S += red[k];
    const int32_t eb = avg_estimate_exp(S);
    crec[c].ebase = eb;
    for (int g = 0; g < ns; ++g) {
      seb[g] = avg_sub_ebase(eb, S);
      S += ssum[s0 + g];
    }
  }
  __syncthreads();
  const int g = t / kAvgHyps, h = t - g * kAvgHyps;
  if (g < ns) {
    const int64_t e0 = (s0 + g) * kAvgSub;
    const AvgHyp r = avg_simulate_hyp(m + e0, (int)min((int64_t)kAvgSub, n - e0), seb[g], h);
    sh[g][h] = r;
    srec[s0 + g].h[h] = r;
    if (h == 0) srec[s0 + g].ebase = seb[g];
  }
  __syncthreads();
  if (t < kAvgHyps) {
    AvgHyp acc = sh[0][t];
    for (int k = 1; k < ns; ++k) acc = avg_compose(acc, t & 1, sh[k][t & ~1], sh[k][t | 1]);
    crec[c].h[t] = acc;
  }
}

// the combine walk, one warp: every lane runs the same sequence on the same (shared-memory) values, so the state and the
// branches are warp-uniform and all lanes help stage the records and data a branch needs
__global__ void __launch_bounds__(32) avg_walk_kernel(const float *__restrict__ m, int64_t n, const AvgRec *__restrict__ srec,
                                                      const AvgRec *__restrict__ crec, float *__restrict__ avg) {
  __shared__ AvgRec cr[32], sr[kAvgGroup];
  __shared__ float xs[kAvgSub];
  const int lane = threadIdx.x;
  const int64_t nsub = ceil_div64(n, kAvgSub);
  const int nch = (int)ceil_div64(nsub, kAvgGroup);
  float a = 0.f;
  for (int c0 = 0; c0 < nch; c0 += 32) {
    __syncwarp();
    if (c0 + lane < nch) cr[lane] = crec[c0 + lane];
    __syncwarp();
    const int c1 = min(nch, c0 + 32);
    for (int c = c0; c < c1; ++c) {
      float j;
      if (avg_try_jump(a, cr[c - c0], &j)) { a = j; continue; }
      const int64_t s0 = (int64_t)c * kAvgGroup;
      const int ns = (int)min((int64_t)kAvgGroup, nsub - s0);
      __syncwarp();
      if (lane < ns) sr[lane] = srec[s0 + lane];
      __syncwarp();
      for (int g = 0; g < ns; ++g) {
        if (avg_try_jump(a, sr[g], &j)) { a = j; continue; }
        const int64_t e0 = (s0 + g) * kAvgSub;
        const int len = (int)min((int64_t)kAvgSub, n - e0);
        __syncwarp();
        for (int i = lane; i < len; i += 32) xs[i] = __ldg(m + e0 + i);
        __syncwarp();
#pragma unroll 8
        for (int i = 0; i < len; ++i) a = __fadd_rn(a, xs[i]);
      }
    }
  }
  if (lane == 0) *avg = avg_finish(a, n);
}

static int launch_exact_avg(const float *m, int64_t n, void *ws, float *avg, cudaStream_t st) {
  const AvgWs w = avg_ws(ws, n);
  avg_sum_kernel<<<w.nch, 256, 0, st>>>(m, n, w.ssum, w.csum);
  FAV_TRY(post_launch("avg.sum"));
  avg_hyp_kernel<<<w.nch, kAvgHypThreads, 0, st>>>(m, n, w.ssum, w.csum, w.srec, w.crec);
  FAV_TRY(post_launch("avg.hyp"));
  avg_walk_kernel<<<1, 32, 0, st>>>(m, n, w.srec, w.crec, avg);
  return post_launch("avg.walk");
}

// fav_compute_corners with the image planes scaled by `scale` (see structure_tensor_kernel)
int launch_compute_corners(const float *image, float scale, int Z, int W, int H, float rho, float *corners, float *avg_out,
                           void *workspace, cudaStream_t st);

}  // namespace fav

using namespace fav;

extern "C" {

int fav_consistency_check(const float *flow1, const float *flow2, const float *structure, float structure_avg,
                          uint8_t *reliable_u8, float *cert_f32, int W, int H, void *stream) {
  FAV_REQUIRE(flow1 && flow2, "consistencyChecker: null flow");
  FAV_REQUIRE(reliable_u8 || cert_f32, "consistencyChecker: no output tensor");
  FAV_REQUIRE(W > 0 && H > 0, "consistencyChecker: empty flow");
  FAV_TRY(require_device());
  const int64_t HW = (int64_t)H * W;
  return launch_consistency(flow1, flow1 + HW, flow2, flow2 + HW, structure, nullptr, structure_avg, reliable_u8,
                            cert_f32, W, H, (cudaStream_t)stream);
}

size_t fav_compute_corners_workspace(int Z, int W, int H) {
  (void)Z;
  // dxx,dyy,dxy + 3 scratch planes + 3 transposed planes + minmax + the per-block maxima / carries / minima of the normalize scan
  // + the chunk sums and records of the exact average (launch_exact_avg), after the normalize scan's area
  const size_t nb = ((size_t)W * H + 1023) / 1024;
  return (size_t)9 * W * H * sizeof(float) + (8 + 3 * nb + 8) * sizeof(float) + 256 + avg_ws_bytes((int64_t)W * H);
}

int fav_compute_corners(const float *image, int Z, int W, int H, float rho, float *corners, float *avg_out,
                        void *workspace, void *stream) {
  FAV_REQUIRE(image && corners && workspace, "computeCorners: null tensor");
  FAV_REQUIRE(Z > 0 && W >= 3 && H >= 3, "computeCorners: image too small");
  FAV_TRY(require_device());
  return launch_compute_corners(image, 1.0f, Z, W, H, rho, corners, avg_out, workspace, (cudaStream_t)stream);
}
}

int fav::launch_compute_corners(const float *image, float scale, int Z, int W, int H, float rho, float *corners, float *avg_out,
                                void *workspace, cudaStream_t st) {
  int64_t n = (int64_t)W * H;
  float *dxx = (float *)workspace, *dyy = dxx + n, *dxy = dyy + n, *scr = dxy + n, *minmax = scr + 6 * n;
  dim3 b2(32, 8), g2(ceil_div(W, 32), ceil_div(H, 8));
  structure_tensor_kernel<<<g2, b2, 0, st>>>(image, scale, Z, W, H, dxx, dyy, dxy);
  FAV_TRY(post_launch("computeCorners.structure"));
  // coefficients exactly as CFilter.h:1420-1426 (double expressions rounded to float)
  IirC c;
  float alpha = (float)(2.5 / (sqrt(3.1415926535897932384626433832795) * (double)rho));
  float e = (float)exp(-(double)alpha);
  c.e2 = e * e;
  c.te = (float)(2.0 * (double)e);
  c.k = (float)((1.0 - (double)e) * (1.0 - (double)e) / (1.0 + 2.0 * (double)alpha * (double)e - (double)c.e2));
  c.pm = (float)((double)e * ((double)alpha - 1.0));
  c.pp = (float)((double)e * ((double)alpha + 1.0));
  // X: one thread per row (stride 1, pitch W); Y: one thread per column (stride W, pitch 1)
  // X pass: lines = rows.  Run it on the transposed matrices (coalesced), transpose back.
  float *tr = scr + 3 * n;
  transpose3_kernel<<<dim3(ceil_div(W, 32), ceil_div(H, 32), 3), 256, 0, st>>>(dxx, tr, H, W, n);
  FAV_TRY(post_launch("computeCorners.transpose"));
  iir_kernel<<<dim3(ceil_div(H, 128), 3), 128, 0, st>>>(tr, tr + n, tr + 2 * n, scr, W, H, H, 1, n, c);
  FAV_TRY(post_launch("computeCorners.iirX"));
  transpose3_kernel<<<dim3(ceil_div(H, 32), ceil_div(W, 32), 3), 256, 0, st>>>(tr, dxx, W, H, n);
  FAV_TRY(post_launch("computeCorners.transposeBack"));
  iir_kernel<<<dim3(ceil_div(W, 128), 3), 128, 0, st>>>(dxx, dyy, dxy, scr, H, W, W, 1, n, c);
  FAV_TRY(post_launch("computeCorners.iirY"));
  eigen_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(dxx, dxy, dyy, corners, n);
  FAV_TRY(post_launch("computeCorners.eigen"));
  {  // normalize(0,1): min / max with the reference's `else if` scan, evaluated as an exact parallel prefix-maximum scan
    const int nb = (int)ceil_div64(n, kNormBlock);
    float *bmax = minmax + 8, *carry = bmax + nb, *bmin = carry + nb + 1;
    norm_block_max_kernel<<<nb, kNormBlock, 0, st>>>(corners, n, bmax);
    FAV_TRY(post_launch("normalize.blockmax"));
    norm_carry_kernel<<<1, 1024, 0, st>>>(bmax, nb, carry);
    FAV_TRY(post_launch("normalize.carry"));
    norm_block_min_kernel<<<nb, kNormBlock, 0, st>>>(corners, n, carry, bmin);
    FAV_TRY(post_launch("normalize.blockmin"));
    norm_final_kernel<<<1, 1024, 0, st>>>(bmin, nb, carry, minmax);
    FAV_TRY(post_launch("normalize.final"));
  }
  normalize_apply_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(corners, n, minmax);
  FAV_TRY(post_launch("normalize.apply"));
  if (avg_out) {
    const size_t nb = (size_t)ceil_div64(n, kNormBlock);
    FAV_TRY(launch_exact_avg(corners, n, (char *)(minmax + 8 + 3 * nb + 8) + 256, avg_out, st));
  }
  return FAV_OK;
}
