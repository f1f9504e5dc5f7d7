// fav_common.cuh -- shared helpers for libfav_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <string>

#include "../../include/fav.h"

namespace fav {

void set_error(const char *fmt, ...);
extern std::atomic<uint64_t> g_launches;

inline int check_cuda(cudaError_t e, const char *what) {
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return FAV_ERR_CUDA;
  }
  return FAV_OK;
}

// after every launch: mirrors the reference's cudaGetLastError() check (BilinearSamplerBDHW.cu:146-150)
inline int post_launch(const char *name) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_cuda(cudaGetLastError(), name);
}

int require_device();  // FAV_ERR_NO_DEVICE when no GPU: there is no CPU fallback

#define FAV_TRY(expr)                 \
  do {                                \
    int _st = (expr);                 \
    if (_st != FAV_OK) return _st;    \
  } while (0)

#define FAV_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      fav::set_error(__VA_ARGS__);    \
      return FAV_ERR_INVALID;         \
    }                                 \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

#ifdef __CUDACC__
// The bilinear blend of BilinearSamplerBDHW.cu:103-106 exactly as nvcc (12.9, default -fmad=true, sm_90a) compiles the
// reference kernel: the TR product is rounded, every other term is fused into the running sum (SASS: FMUL,FMUL,FMUL,FFMA,
// FMUL,FMUL,FFMA,FFMA).  Pinned bit-for-bit against the reference's own kernel body compiled from /root/reference
// (oracle/ref_warp/, tests/test_gpu_refwarp.py).  wx, wy = weights of the top-left corner, omx = 1 - wx, omy = 1 - wy.
__device__ __forceinline__ float bilinear_ref_blend(float wx, float wy, float omx, float omy, float vtl, float vtr,
                                                    float vbl, float vbr) {
  float v = __fmul_rn(__fmul_rn(omx, wy), vtr);
  v = __fmaf_rn(__fmul_rn(wx, wy), vtl, v);
  v = __fmaf_rn(__fmul_rn(wx, omy), vbl, v);
  return __fmaf_rn(__fmul_rn(omx, omy), vbr, v);
}
#endif

// VGG mean, BGR order (fast_artistic_video/preprocess.lua:48)
#define FAV_MEAN_B 103.939f
#define FAV_MEAN_G 116.779f
#define FAV_MEAN_R 123.68f

}  // namespace fav
