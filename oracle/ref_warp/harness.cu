// oracle/ref_warp/harness.cu -- TEST INFRASTRUCTURE ONLY (the pin of the warp oracle and the "kernel to beat").
//
// Wraps the reference's own CUDA kernel BilinearSamplerBDHW_bilinearSamplingFromGrid in a plain C entry point.
// The kernel body is NOT in this repository: oracle/Makefile extracts lines 6-32 (stride_t + device helpers) and 48-109
// (the __global__ kernel) of /root/reference/stnbdhw/BilinearSamplerBDHW.cu into oracle/_ref/ref_warp_kernel.inc at
// build time and compiles this file for sm_90a with nvcc's default flags (the reference's CMakeLists.txt:55 adds only
// an -arch flag, so FMA contraction is on, as here).  The launch configuration below is the reference launcher's
// (BilinearSamplerBDHW.cu:119-120): blocks (C, Hout * ceil(Wout / 512), B), threads (32, 16).
#include <cuda_runtime.h>
#include <stdint.h>

#include "ref_warp_kernel.inc"

extern "C" __attribute__((visibility("default"))) int ref_warp_bdhw_update_output(
    const float *img, const int isz[4], const int ist[4], const float *grid, const int gst[4], float *out,
    const int ost[4], int Hout, int Wout, void *stream) {
  dim3 blocks(isz[1], Hout * ((Wout + 511) / 512), isz[0]);  // :119
  dim3 threads(32, 16);                                      // :120
  BilinearSamplerBDHW_bilinearSamplingFromGrid<<<blocks, threads, 0, (cudaStream_t)stream>>>(
      const_cast<float *>(img), stride_t{ist[0], ist[1], ist[2], ist[3]}, const_cast<float *>(grid),
      stride_t{gst[0], gst[1], gst[2], gst[3]}, out, stride_t{ost[0], ost[1], ost[2], ost[3]}, isz[1], isz[2], isz[3], Hout,
      Wout);
  return (int)cudaGetLastError();  // :146-150
}
