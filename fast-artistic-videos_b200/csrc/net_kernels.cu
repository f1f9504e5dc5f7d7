// net_kernels.cu -- HBM-bound kernels of the stylization net + the CUDA-core convolution comparator.
//   pack_input      : fp32 NCHW net input -> (reflect-padded) fp16 hi/lo operand     train_video.lua:319-324
//   in_stats        : per-channel sum / sum of squares of a raw conv output         InstanceNormalization.lua:33-53
//   in_finalize     : mean, gamma/sqrt(var+eps), beta (biased variance, eps 1e-5)
//   in_apply        : normalise (+ReLU) (+ShaveImage(2) skip add) -> next operand    models_video.lua:41-53,121-130
//   unpack_operand  : operand -> fp32 NCHW (per-layer parity checks)
//   conv_simt       : direct convolution on CUDA cores, same I/O as the tcgen05 kernel (bring-up comparator)
#include "conv.cuh"

namespace fav {

constexpr int kStatRows = 8;
constexpr int kApplyIter = 4;  // pixels per thread in the apply kernels: amortises the per-block finalisation

__device__ __forceinline__ void load_join8(const uint4 *hi_src, const uint4 *lo_src, float v[8]) {
  uint4 h = __ldg(hi_src), l = __ldg(lo_src);
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __half2float(__ushort_as_half((unsigned short)(hw[i] & 0xffff))) +
               __half2float(__ushort_as_half((unsigned short)(lw[i] & 0xffff)));
    v[2 * i + 1] = __half2float(__ushort_as_half((unsigned short)(hw[i] >> 16))) +
                   __half2float(__ushort_as_half((unsigned short)(lw[i] >> 16)));
  }
}

// ---- pack_input --------------------------------------------------------------------------------------
// in: [Cin][H][W] fp32.  dst logical size = (H+2R) x (W+2R) with R = reflect (nn.SpatialReflectionPadding:
// index -i for i<0, 2(n-1)-i for i>=n).  One thread per (padded pixel, channel block).
__global__ void __launch_bounds__(256) pack_input_kernel(const float *__restrict__ in, int Cin, int H, int W, int R,
                                                         Operand dst) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  int cb = blockIdx.z;
  if (x >= dst.W) return;
  int sy = y - R, sx = x - R;
  sy = sy < 0 ? -sy : (sy >= H ? 2 * (H - 1) - sy : sy);
  sx = sx < 0 ? -sx : (sx >= W ? 2 * (W - 1) - sx : sx);
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = cb * 8 + i;
    v[i] = c < Cin ? __ldg(in + ((int64_t)c * H + sy) * W + sx) : 0.f;
  }
  int64_t o = dst.off16(dst.padT + y, cb, dst.padL + x);
  split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
}

int launch_pack_input(const float *in, int Cin, int H, int W, int reflect, const Operand &dst, cudaStream_t st) {
  dim3 grid(ceil_div(dst.W, 256), dst.H, dst.Cb);
  pack_input_kernel<<<grid, 256, 0, st>>>(in, Cin, H, W, reflect, dst);
  return post_launch("pack_input");
}

// ---- in_stats ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) in_stats_kernel(RawTensor raw, double *__restrict__ sums) {
  const int cq = blockIdx.x;
  const int y0 = blockIdx.y * kStatRows;
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  for (int y = y0; y < min(y0 + kStatRows, raw.H); ++y) {
    const float4 *row = reinterpret_cast<const float4 *>(raw.p) + raw.off4(y, cq, 0);
    for (int x = threadIdx.x; x < raw.W; x += 256) {
      float4 v;
      if (raw.planar) {
        v.x = cq * 4 + 0 < raw.C ? __ldg(raw.p + raw.offp(cq * 4 + 0, y, x)) : 0.f;
        v.y = cq * 4 + 1 < raw.C ? __ldg(raw.p + raw.offp(cq * 4 + 1, y, x)) : 0.f;
        v.z = cq * 4 + 2 < raw.C ? __ldg(raw.p + raw.offp(cq * 4 + 2, y, x)) : 0.f;
        v.w = cq * 4 + 3 < raw.C ? __ldg(raw.p + raw.offp(cq * 4 + 3, y, x)) : 0.f;
      } else
      v = __ldg(row + x);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
      q[0] += v.x * v.x; q[1] += v.y * v.y; q[2] += v.z * v.z; q[3] += v.w * v.w;
    }
  }
  __shared__ double red[8][8];
  double d[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) { d[i] = s[i]; d[4 + i] = q[i]; }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d[i] += __shfl_xor_sync(0xffffffffu, d[i], o);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][i] = d[i];
  __syncthreads();
  if (threadIdx.x < 8) {
    double t = 0;
    for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
    int i = threadIdx.x & 3;
    int c = cq * 4 + i;
    if (c < raw.C) atomicAdd(sums + (threadIdx.x < 4 ? c : raw.C + c), t);
  }
}

int launch_in_stats(const RawTensor &raw, double *sums, cudaStream_t st) {
  dim3 grid(raw.Cq, ceil_div(raw.H, kStatRows));
  in_stats_kernel<<<grid, 256, 0, st>>>(raw, sums);
  return post_launch("in_stats");
}

// ---- in_apply ----------------------------------------------------------------------------------------
// mean / gamma*rstd / beta of the block's 8 channels are derived from the (double) sums by the first 8 threads:
// biased variance, eps inside the sqrt (nn.SpatialBatchNormalization in training mode, InstanceNormalization.lua:39-50)
template <int ITER>
__global__ void __launch_bounds__(128) in_apply_kernel(RawTensor raw, const double *__restrict__ sums,
                                                       const float *__restrict__ gamma, const float *__restrict__ beta,
                                                       double inv_count, double eps, int relu, Operand skip, int has_skip,
                                                       int shave, Operand dst) {
  __shared__ float s_mean[8], s_scale[8], s_beta[8];
  const int xbase = blockIdx.x * (128 * ITER) + threadIdx.x;
  const int y = blockIdx.y, cb = blockIdx.z;
  // 1. every streaming load of the thread is requested first (they do not depend on the statistics): the per-block
  //    finalisation below (dependent global loads + double sqrt / divide on 8 threads) then runs in their shadow
  float v[ITER][8];
  uint4 skh[ITER], skl[ITER];
  const float4 *rp = reinterpret_cast<const float4 *>(raw.p);
#pragma unroll
  for (int it = 0; it < ITER; ++it) {
    const int x = xbase + it * 128;
    if (x < raw.W) {
      if (raw.planar) {  // planar raw tensor: one plane per channel, lanes run along x (128-byte coalesced per plane)
        const float *p0 = raw.p + raw.offp(cb * 8, y, x);
        const int64_t plane = (int64_t)raw.Hp * raw.Wp;
#pragma unroll
        for (int i = 0; i < 8; ++i) v[it][i] = __ldg(p0 + i * plane);
      } else {
        const float4 a = __ldg(rp + raw.off4(y, 2 * cb, x)), b = __ldg(rp + raw.off4(y, 2 * cb + 1, x));
        v[it][0] = a.x; v[it][1] = a.y; v[it][2] = a.z; v[it][3] = a.w; v[it][4] = b.x; v[it][5] = b.y; v[it][6] = b.z; v[it][7] = b.w;
      }
      if (has_skip) {  // ConcatTable{conv_block, ShaveImage(2)} -> CAddTable (models_video.lua:41-53)
        const int64_t so = skip.off16(skip.padT + y + shave, cb, skip.padL + x + shave);
        skh[it] = __ldg(reinterpret_cast<const uint4 *>(skip.hi) + so);
        skl[it] = __ldg(reinterpret_cast<const uint4 *>(skip.lo) + so);
      }
    }
  }
  // 2. mean / gamma * rstd / beta of the block's 8 channels
  if (threadIdx.x < 8) {
    int c = cb * 8 + threadIdx.x;
    in_finalize(sums[c], sums[raw.C + c], inv_count, eps, gamma[c], s_mean[threadIdx.x], s_scale[threadIdx.x]);
    s_beta[threadIdx.x] = beta[c];
  }
  __syncthreads();
  // 3. normalise (+ReLU) (+skip), split into fp16 hi / lo, store the next operand
#pragma unroll
  for (int it = 0; it < ITER; ++it) {
    const int x = xbase + it * 128;
    if (x >= raw.W) break;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float t = (v[it][i] - s_mean[i]) * s_scale[i] + s_beta[i];
      v[it][i] = relu ? fmaxf(t, 0.f) : t;
    }
    if (has_skip) {
      const uint32_t hw[4] = {skh[it].x, skh[it].y, skh[it].z, skh[it].w}, lw[4] = {skl[it].x, skl[it].y, skl[it].z, skl[it].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {  // same arithmetic as load_join8
        v[it][2 * i] += __half2float(__ushort_as_half((unsigned short)(hw[i] & 0xffff))) +
                        __half2float(__ushort_as_half((unsigned short)(lw[i] & 0xffff)));
        v[it][2 * i + 1] += __half2float(__ushort_as_half((unsigned short)(hw[i] >> 16))) +
                            __half2float(__ushort_as_half((unsigned short)(lw[i] >> 16)));
      }
    }
    const int64_t o = dst.off16(dst.padT + y, cb, dst.padL + x);
    split_store8(v[it], reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
  }
}

int launch_in_apply(const RawTensor &raw, const double *sums, const float *gamma, const float *beta, float eps, int relu,
                    const Operand *skip, int shave, const Operand &dst, cudaStream_t st) {
  // pixels per thread: amortises the per-block finalisation against registers (occupancy); FAV_APPLY_ITER = 2|3|4 for A/B timing
  static const int forced = getenv("FAV_APPLY_ITER") ? atoi(getenv("FAV_APPLY_ITER")) : 0;
  const int iter = forced >= 2 && forced <= 4 ? forced : kApplyIter;
  dim3 grid(ceil_div(raw.W, 128 * iter), raw.H, raw.C / 8);
  Operand sk = skip ? *skip : Operand();
  const double inv = 1.0 / ((double)raw.H * raw.W);
  if (iter == 2)
    in_apply_kernel<2><<<grid, 128, 0, st>>>(raw, sums, gamma, beta, inv, (double)eps, relu, sk, skip ? 1 : 0, shave, dst);
  else if (iter == 3)
    in_apply_kernel<3><<<grid, 128, 0, st>>>(raw, sums, gamma, beta, inv, (double)eps, relu, sk, skip ? 1 : 0, shave, dst);
  else
    in_apply_kernel<4><<<grid, 128, 0, st>>>(raw, sums, gamma, beta, inv, (double)eps, relu, sk, skip ? 1 : 0, shave, dst);
  return post_launch("in_apply");
}

// (Tried and removed, DESIGN.md 9: a streaming version of in_apply -- persistent blocks, one producer thread feeding a 3-stage
// shared-memory ring with cp.async.bulk row copies, 8 consumer warps -- on the theory that the kernel is latency bound by its
// register-held loads.  Measured: residual layers 20.8 us vs 21-23 us, wide layers SLOWER (53.6 vs 50.0, 47.5 vs 41.2 us),
// 915 vs 924 frames/s.  Neither the issue slots (packed conversions: -35 % instructions, same time) nor the loads in flight
// bound this kernel.)

// ---- nn.SpatialUpSamplingNearest(s) -> InstanceNormalization -> ReLU on an OPERAND (arch token UX) ---------------
// models_video.lua:94-98,121-130.  Statistics of a nearest-upsampled tensor equal those of its source, so the sums
// are taken over the source operand and the upsampling happens while the normalised values are written.
__global__ void __launch_bounds__(256) opnd_stats_kernel(Operand src, double *__restrict__ sums) {
  const int cb = blockIdx.x;
  const int y0 = blockIdx.y * kStatRows;
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = 0.f;
  for (int y = y0; y < min(y0 + kStatRows, src.H); ++y)
    for (int x = threadIdx.x; x < src.W; x += 256) {
      float v[8];
      int64_t o = src.off16(src.padT + y, cb, src.padL + x);
      load_join8(reinterpret_cast<const uint4 *>(src.hi) + o, reinterpret_cast<const uint4 *>(src.lo) + o, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] += v[i]; q[i] += v[i] * v[i]; }
    }
  __shared__ double red[8][16];
  double d[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) { d[i] = s[i]; d[8 + i] = q[i]; }
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d[i] += __shfl_xor_sync(0xffffffffu, d[i], o);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < 16; ++i) red[warp][i] = d[i];
  __syncthreads();
  if (threadIdx.x < 16) {
    double t = 0;
    for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
    int c = cb * 8 + (threadIdx.x & 7);
    if (c < src.C) atomicAdd(sums + (threadIdx.x < 8 ? c : src.C + c), t);
  }
}

__global__ void __launch_bounds__(128) up_apply_kernel(Operand src, const double *__restrict__ sums,
                                                       const float *__restrict__ gamma, const float *__restrict__ beta,
                                                       double inv_count, double eps, int relu, int scale, Operand dst) {
  __shared__ float s_mean[8], s_scale[8], s_beta[8];
  const int xbase = blockIdx.x * (128 * kApplyIter) + threadIdx.x;
  const int y = blockIdx.y, cb = blockIdx.z;
  if (threadIdx.x < 8) {
    int c = cb * 8 + threadIdx.x;
    in_finalize(sums[c], sums[src.C + c], inv_count, eps, gamma[c], s_mean[threadIdx.x], s_scale[threadIdx.x]);
    s_beta[threadIdx.x] = beta[c];
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kApplyIter; ++it) {
    const int x = xbase + it * 128;
    if (x >= dst.W) return;
    float v[8];
    int64_t so = src.off16(src.padT + y / scale, cb, src.padL + x / scale);
    load_join8(reinterpret_cast<const uint4 *>(src.hi) + so, reinterpret_cast<const uint4 *>(src.lo) + so, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float t = (v[i] - s_mean[i]) * s_scale[i] + s_beta[i];
      v[i] = relu ? fmaxf(t, 0.f) : t;
    }
    int64_t o = dst.off16(dst.padT + y, cb, dst.padL + x);
    split_store8(v, reinterpret_cast<uint4 *>(dst.hi) + o, reinterpret_cast<uint4 *>(dst.lo) + o);
  }
}

int launch_up_in(const Operand &src, double *sums, const float *gamma, const float *beta, float eps, int relu, int scale,
                 const Operand &dst, cudaStream_t st) {
  opnd_stats_kernel<<<dim3(src.Cb, ceil_div(src.H, kStatRows)), 256, 0, st>>>(src, sums);
  FAV_TRY(post_launch("up_in.stats"));
  dim3 grid(ceil_div(dst.W, 128 * kApplyIter), dst.H, dst.Cb);
  up_apply_kernel<<<grid, 128, 0, st>>>(src, sums, gamma, beta, 1.0 / ((double)src.H * src.W), (double)eps, relu, scale, dst);
  return post_launch("up_in.apply");
}

// ---- unpack_operand (debug) -----------------------------------------------------------------------------
__global__ void __launch_bounds__(128) unpack_kernel(Operand src, float *__restrict__ out) {
  int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y, cb = blockIdx.z;
  if (x >= src.W) return;
  float v[8];
  int64_t o = src.off16(src.padT + y, cb, src.padL + x);
  load_join8(reinterpret_cast<const uint4 *>(src.hi) + o, reinterpret_cast<const uint4 *>(src.lo) + o, v);
  for (int i = 0; i < 8; ++i) {
    int c = cb * 8 + i;
    if (c < src.C) out[((int64_t)c * src.H + y) * src.W + x] = v[i];
  }
}
int launch_unpack_operand(const Operand &src, float *out, cudaStream_t st) {
  dim3 grid(ceil_div(src.W, 128), src.H, src.Cb);
  unpack_kernel<<<grid, 128, 0, st>>>(src, out);
  return post_launch("unpack_operand");
}

// ---- conv_simt: CUDA-core direct convolution (comparator) ---------------------------------------------------
// block = 128 threads = 128 consecutive output pixels of one row; blockIdx.y = output row; blockIdx.z = group of
// 8 output channels.  fp32 FMA over (hi + lo) activations and fp32 weights.
__device__ __forceinline__ float final_value(float v, int k, int mode, float tanh_c) {
  float t = tanhf(v) * tanh_c;  // nn.Tanh -> nn.MulConstant (models_video.lua:135-136)
  if (mode == 2) {              // fused vgg.deprocess (preprocess.lua:70)
    const float mean[3] = {FAV_MEAN_B, FAV_MEAN_G, FAV_MEAN_R};
    t = __fdiv_rn(__fadd_rn(t, mean[k]), 255.0f);
  }
  return t;
}

__global__ void __launch_bounds__(128) conv_simt_kernel(const __grid_constant__ SimtJob j) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int co0 = blockIdx.z * 8;
  if (x >= j.Wo) return;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const uint4 *hi = reinterpret_cast<const uint4 *>(j.in.hi), *lo = reinterpret_cast<const uint4 *>(j.in.lo);
  for (int t = 0; t < j.ntaps; ++t) {
    int ys = j.in.padT + j.sy * y + j.tdy[t], xs = j.in.padL + j.sx * x + j.tdx[t];
    for (int cb = 0; cb < j.in.Cb; ++cb) {
      float a[8];
      int64_t o = j.in.off16(ys, cb, xs);
      load_join8(hi + o, lo + o, a);
      const float *w = j.w + ((int64_t)t * j.Cin_pad + cb * 8) * j.Cout_pad8 + co0;
#pragma unroll
      for (int ci = 0; ci < 8; ++ci) {
        float4 w0 = __ldg(reinterpret_cast<const float4 *>(w + (int64_t)ci * j.Cout_pad8));
        float4 w1 = __ldg(reinterpret_cast<const float4 *>(w + (int64_t)ci * j.Cout_pad8 + 4));
        acc[0] = fmaf(a[ci], w0.x, acc[0]); acc[1] = fmaf(a[ci], w0.y, acc[1]);
        acc[2] = fmaf(a[ci], w0.z, acc[2]); acc[3] = fmaf(a[ci], w0.w, acc[3]);
        acc[4] = fmaf(a[ci], w1.x, acc[4]); acc[5] = fmaf(a[ci], w1.y, acc[5]);
        acc[6] = fmaf(a[ci], w1.z, acc[6]); acc[7] = fmaf(a[ci], w1.w, acc[7]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] += (co0 + i < j.Cout) ? __ldg(j.bias + co0 + i) : 0.f;
  const int yo = y * j.oy_mul + j.oy_off, xo = x * j.ox_mul + j.ox_off;
  if (j.final_mode == 0 && j.raw_planar) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (co0 + i < j.Cout) j.raw[((int64_t)(co0 + i) * j.raw_Hp + yo) * j.raw_Wp + xo] = acc[i];
  } else if (j.final_mode == 0) {
    float4 *rp = reinterpret_cast<float4 *>(j.raw);
    int64_t o0 = (((int64_t)yo * j.raw_Cq + (co0 >> 2)) * j.raw_Wp + xo);
    rp[o0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    if ((co0 >> 2) + 1 < j.raw_Cq) rp[o0 + j.raw_Wp] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  } else {
    for (int k = 0; k < 8; ++k)
      if (co0 + k < j.Cout)
        j.out3[((int64_t)(j.final_mode == 2 ? 2 - (co0 + k) : co0 + k) * j.Ho + yo) * j.Wo + xo] =
            final_value(acc[k], co0 + k, j.final_mode, j.tanh_c);
  }
}

int launch_conv_simt(const SimtJob &job, cudaStream_t st) {
  dim3 grid(ceil_div(job.Wo, 128), job.Ho, job.Cout_pad8 / 8);
  conv_simt_kernel<<<grid, 128, 0, st>>>(job);
  return post_launch("conv_simt");
}

}  // namespace fav
