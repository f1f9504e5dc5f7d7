// exact_avg.cuh -- CMatrix::avg (CMatrix.h:1245-1251) evaluated in parallel, bit-identical to the sequential fp32 chain
//   a_0 = +0,  a_{k+1} = fl(a_k + x_k),  avg = fl(a_n / (float)n).
// Shared by the kernels of consistency.cu and the CPU emulator tests/emu/avg_emu.cu.
//
// Why a parallel evaluation can be exact.  Let a have exponent E (2^E <= |a| < 2^(E+1)) and u = 2^(E-23), so a = M u with M an
// integer, 2^23 <= |M| < 2^24.  While the exact a + x stays in that binade with the same sign, fl(a + x) = (M + q) u where q is
// x/u (exact in double) rounded to the nearest integer, a tie going to the even M + q.  Within a run of such steps the chain is
// an integer sum that depends on its start only through (E, parity of M) and on staying inside the binade.  So:
//   1. the data is cut into sub-chunks of kAvgSub elements and chunks of kAvgGroup sub-chunks;
//   2. for each sub-chunk and each hypothesis h = (E, parity) one thread runs the sub-chunk in integers (avg_simulate) and
//      records the offset d and the minimum / maximum of the running offset; a chunk's records are its sub-chunks' records
//      composed in order (avg_compose).  E in {Ê - 1, Ê, Ê + 1}, Ê the exponent of a double prefix sum of the data before the
//      chunk: for data of one sign the fp32 chain stays within a factor (1 +- 2^-24)^n of that sum, inside those three binades
//      up to n ~ 2^23.  The estimate only decides which hypotheses are precomputed, it never changes a bit;
//   3. the chunks are combined in order from the exact state: the chunk's record for the state's (E, parity) applies when the
//      running |M| stays inside [2^23 + 1, 2^24 - 1] (then every exact partial sum lies in [2^23 + 1/2, 2^24 - 1/2] u, where
//      the fp32 grid is the integers times u), and the state jumps by d (avg_try_jump).  Otherwise the chunk's sub-chunks are
//      combined the same way, and a sub-chunk without an applicable record runs its kAvgSub FADDs.  The first elements (small
//      |a|), the ~log2 n binade crossings, cancellation across zero (values may be negative: CMatrix::normalize's `else if`
//      quirk) and NaN / Inf take the FADD branch.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

namespace fav {

constexpr int kAvgSub = 256;                      // elements per sub-chunk
constexpr int kAvgGroup = 32;                     // sub-chunks per chunk (one warp lane each in the combine walk)
constexpr int kAvgChunk = kAvgSub * kAvgGroup;    // elements per chunk
constexpr int kAvgHyps = 6;                       // E in {Ê-1, Ê, Ê+1} x parity of M
constexpr int32_t kAvgNoEstimate = INT32_MIN;     // no precomputed hypotheses (estimate 0, subnormal or not finite)
constexpr int32_t kAvgBad = -(1 << 30);           // AvgHyp::dmin of a hypothesis that leaves every binade window

struct AvgHyp { int32_t d, dmin, dmax; };         // offset of M over the run, min / max of the running offset (including 0)
struct AvgRec { int32_t ebase; AvgHyp h[kAvgHyps]; };  // h[2 j + p]: E = ebase + j - 1, parity p

__host__ __device__ inline AvgHyp avg_bad() { return AvgHyp{0, kAvgBad, -kAvgBad}; }
__host__ __device__ inline bool avg_ok(const AvgHyp &h) { return h.dmin > kAvgBad; }

__host__ __device__ inline float avg_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline uint32_t avg_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
  return b;
#endif
}
__host__ __device__ inline float avg_float(uint32_t b) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}

// Ê of a double estimate of the running sum; kAvgNoEstimate where no fp32 state of a normal binade is expected
__host__ __device__ inline int32_t avg_estimate_exp(double s) {
  s = fabs(s);
  if (!(s >= 0x1p-126 && s < 0x1p128)) return kAvgNoEstimate;
  int e;
  frexp(s, &e);
  return e - 1;
}

// one hypothesis (E, parity) over len elements, in integers
__host__ __device__ inline AvgHyp avg_simulate(const float *x, int len, int E, int parity) {
  const double scale = ldexp(1.0, 23 - E);
  int32_t d = 0, lo = 0, hi = 0;
  for (int k = 0; k < len; ++k) {
    const double t = (double)x[k] * scale;  // exact: a float times a power of two, far from the double range's ends
    if (!(fabs(t) < 0x1p25)) return avg_bad();  // also NaN / Inf
    const double f = floor(t);
    int32_t q = (int32_t)f;
    const double r = t - f;  // exact
    if (r > 0.5 || (r == 0.5 && ((parity + d + q) & 1))) ++q;  // nearest, the tie to the even M + q
    d += q;
    lo = d < lo ? d : lo;
    hi = d > hi ? d : hi;
    if (lo <= -(1 << 24) || hi >= (1 << 24)) return avg_bad();  // |M| spans less than 2^23: outside every window
  }
  return AvgHyp{d, lo, hi};
}

// hypothesis (E, parity) over a run followed by the next run: the second run starts with the parity parity ^ (acc.d & 1), so
// `next` holds both parities' records of the second run
__host__ __device__ inline AvgHyp avg_compose(const AvgHyp &acc, int parity, const AvgHyp &next0, const AvgHyp &next1) {
  const AvgHyp &n = ((parity + acc.d) & 1) ? next1 : next0;
  if (!avg_ok(acc) || !avg_ok(n)) return avg_bad();
  const int32_t lo = acc.d + n.dmin < acc.dmin ? acc.d + n.dmin : acc.dmin;
  const int32_t hi = acc.d + n.dmax > acc.dmax ? acc.d + n.dmax : acc.dmax;
  if (lo <= -(1 << 24) || hi >= (1 << 24)) return avg_bad();
  return AvgHyp{acc.d + n.d, lo, hi};
}

// the run's record for the state a, if it applies: *out = the state after the run, exactly
__host__ __device__ inline bool avg_try_jump(float a, const AvgRec &r, float *out) {
  if (r.ebase == kAvgNoEstimate) return false;
  const uint32_t b = avg_bits(a);
  const int ef = (int)((b >> 23) & 255);
  if (ef == 0 || ef == 255) return false;  // zero, subnormal, Inf, NaN
  const int j = ef - 127 - r.ebase + 1;
  if (j < 0 || j > 2) return false;
  const int32_t m = (int32_t)((b & 0x7fffffu) | 0x800000u);
  const AvgHyp &h = r.h[2 * j + (m & 1)];
  const bool neg = b >> 31;  // |M| runs as m + D (a > 0) or m - D (a < 0)
  const int64_t lo = neg ? (int64_t)m - h.dmax : (int64_t)m + h.dmin;
  const int64_t hi = neg ? (int64_t)m - h.dmin : (int64_t)m + h.dmax;
  if (!avg_ok(h) || lo < (1 << 23) + 1 || hi > (1 << 24) - 1) return false;
  const uint32_t mag = (uint32_t)(neg ? m - h.d : m + h.d);
  *out = avg_float((b & 0xff800000u) | (mag & 0x7fffffu));
  return true;
}

// the hypotheses of a sub-chunk use its chunk's Ê, so that the chunk's records compose from them; a chunk without an estimate
// (the first one: its prefix sum is 0) lets each sub-chunk use its own
__host__ __device__ inline int32_t avg_sub_ebase(int32_t chunk_ebase, double sub_prefix) {
  return chunk_ebase != kAvgNoEstimate ? chunk_ebase : avg_estimate_exp(sub_prefix);
}

__host__ __device__ inline AvgHyp avg_simulate_hyp(const float *x, int len, int32_t ebase, int h) {
  return ebase == kAvgNoEstimate ? avg_bad() : avg_simulate(x, len, ebase + h / 2 - 1, h & 1);
}

__host__ __device__ inline float avg_finish(float a, int64_t n) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, (float)(int)n);
#else
  return a / (float)(int)n;
#endif
}

}  // namespace fav
