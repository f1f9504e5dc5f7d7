// scale.cu -- image.scale(src, Wout, Hout, 'bicubic') of the `image` rock, as run_image uses it for -scale_factor
// (fast_artistic_video_core.lua:127-129,150-152).
//
// The rock (not vendored, so not pinned here) scales in two separable 1-D passes: every row from Win to Wout into an fp32
// intermediate [C][Hin][Wout], then every column from Hin to Hout.  One pass maps a line of n samples to m:
//   m == n: copy.  Otherwise s = (float)(n-1)/(m-1) and, for d = 0 .. m-2, t = d*s, i = (int)t (<= n-2), f = t - i,
//   p1 = src[i], p2 = src[i+1], p0 = i > 0 ? src[i-1] : 2*p1 - p2, p3 = i+2 < n ? src[i+2] : 2*p2 - p1,
//   dst[d] = p1 + 0.5*f*((p2-p0) + f*((2*p0 - 5*p1 + 4*p2 - p3) + f*(3*(p1-p2) + p3 - p0))); dst[m-1] = src[n-1].
// That is Catmull-Rom (Keys, a = -1/2) on an align-corners grid, with linearly extrapolated borders, no anti-alias prefilter
// when shrinking, and no clamping of the result.
//
// Here both passes are fused: each output pixel takes the x pass of the (up to) four source rows its y taps need, then runs
// the y pass on those four fp32 values.  Every operation is an explicitly rounded fp32 intrinsic in the order above (no FMA
// contraction), so the result is bit-identical to the two-pass form evaluated in fp32.
#include "fav_common.cuh"

namespace fav {

// one sample of the 1-D reading from its four taps
__device__ __forceinline__ float cubic_rn(float p0, float p1, float p2, float p3, float f) {
  const float a1 = __fsub_rn(p2, p0);
  const float a2 = __fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(2.0f, p0), __fmul_rn(5.0f, p1)), __fmul_rn(4.0f, p2)), p3);
  const float a3 = __fsub_rn(__fadd_rn(__fmul_rn(3.0f, __fsub_rn(p1, p2)), p3), p0);
  const float v = __fadd_rn(a1, __fmul_rn(f, __fadd_rn(a2, __fmul_rn(f, a3))));
  return __fadd_rn(p1, __fmul_rn(__fmul_rn(0.5f, f), v));
}

__device__ __forceinline__ float extrapolate_rn(float near, float far) { return __fsub_rn(__fmul_rn(2.0f, near), far); }

// where output sample d of a line of n -> m samples reads: mode 0 copy of src[i], 1 interpolation at i + f
struct LineTap {
  int i, mode;
  float f;
};

__device__ __forceinline__ LineTap line_tap(int d, int n, int m, float s) {
  LineTap t;
  if (m == n) { t.i = d; t.mode = 0; t.f = 0.f; return t; }
  if (d == m - 1) { t.i = n - 1; t.mode = 0; t.f = 0.f; return t; }
  const float pos = __fmul_rn((float)d, s);
  t.i = min((int)pos, n - 2);
  t.f = __fsub_rn(pos, (float)t.i);
  t.mode = 1;
  return t;
}

// the x pass at one output column of source row `row`
__device__ __forceinline__ float x_pass(const float *__restrict__ row, const LineTap &tx, int n) {
  if (tx.mode == 0) return __ldg(row + tx.i);
  const float p1 = __ldg(row + tx.i), p2 = __ldg(row + tx.i + 1);
  const float p0 = tx.i > 0 ? __ldg(row + tx.i - 1) : extrapolate_rn(p1, p2);
  const float p3 = tx.i + 2 < n ? __ldg(row + tx.i + 2) : extrapolate_rn(p2, p1);
  return cubic_rn(p0, p1, p2, p3, tx.f);
}

// one output pixel per thread; blockIdx.z = channel.  sx, sy: the fp32 steps (n-1)/(m-1) of the two passes
__global__ void __launch_bounds__(256) scale_bicubic_kernel(const float *__restrict__ in, float *__restrict__ out, int Hin,
                                                            int Win, int Hout, int Wout, float sx, float sy) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= Wout || y >= Hout) return;
  const float *src = in + (int64_t)blockIdx.z * Hin * Win;
  const LineTap tx = line_tap(x, Win, Wout, sx), ty = line_tap(y, Hin, Hout, sy);
  float v;
  if (ty.mode == 0) {
    v = x_pass(src + (int64_t)ty.i * Win, tx, Win);
  } else {
    const float q1 = x_pass(src + (int64_t)ty.i * Win, tx, Win), q2 = x_pass(src + (int64_t)(ty.i + 1) * Win, tx, Win);
    const float q0 = ty.i > 0 ? x_pass(src + (int64_t)(ty.i - 1) * Win, tx, Win) : extrapolate_rn(q1, q2);
    const float q3 = ty.i + 2 < Hin ? x_pass(src + (int64_t)(ty.i + 2) * Win, tx, Win) : extrapolate_rn(q2, q1);
    v = cubic_rn(q0, q1, q2, q3, ty.f);
  }
  out[((int64_t)blockIdx.z * Hout + y) * Wout + x] = v;
}

constexpr int kScaleMaxSize = 65535;  // (float)d is exact and the grid fits (8 rows per block, one channel per z)

int check_scale_args(const float *in, const float *out, int C, int Hin, int Win, int Hout, int Wout) {
  FAV_REQUIRE(in && out, "image_scale_bicubic: null tensor");
  FAV_REQUIRE(C >= 1 && C <= kScaleMaxSize, "image_scale_bicubic: %d channels (1 to %d)", C, kScaleMaxSize);
  // a line of one sample has no (n-1)/(m-1) step: the rock's branches for it are not pinned, and no frame is that small
  FAV_REQUIRE(Hin >= 2 && Win >= 2 && Hout >= 2 && Wout >= 2 && Hin <= kScaleMaxSize && Win <= kScaleMaxSize &&
                  Hout <= kScaleMaxSize && Wout <= kScaleMaxSize,
              "image_scale_bicubic: %dx%d -> %dx%d: every size must be 2 to %d", Win, Hin, Wout, Hout, kScaleMaxSize);
  return FAV_OK;
}

int launch_image_scale_bicubic(const float *in, float *out, int C, int Hin, int Win, int Hout, int Wout, cudaStream_t st) {
  FAV_TRY(check_scale_args(in, out, C, Hin, Win, Hout, Wout));
  // s = (float)(n-1)/(m-1): one IEEE fp32 division, the same on the host as in the rock
  const float sx = (float)(Win - 1) / (float)(Wout - 1), sy = (float)(Hin - 1) / (float)(Hout - 1);
  dim3 block(32, 8), grid(ceil_div(Wout, 32), ceil_div(Hout, 8), C);
  scale_bicubic_kernel<<<grid, block, 0, st>>>(in, out, Hin, Win, Hout, Wout, sx, sy);
  return post_launch("image_scale_bicubic");
}

}  // namespace fav

using namespace fav;

extern "C" {

int fav_image_scale_bicubic(const float *in, float *out, int C, int Hin, int Win, int Hout, int Wout, void *stream) {
  FAV_TRY(check_scale_args(in, out, C, Hin, Win, Hout, Wout));
  FAV_TRY(require_device());
  return launch_image_scale_bicubic(in, out, C, Hin, Win, Hout, Wout, (cudaStream_t)stream);
}
}
