// conv_tc.cu -- the hot kernel: implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the cuDNN / THNN SpatialConvolution + SpatialFullConvolution calls of the reference net
// (fast_artistic_video/models_video.lua:80,93,102; fast_artistic_video_core.lua:48-55).
//
// GEMM view (per tile):  D[128 pixels, Npad couts] += A[128 pixels, K] * B[Npad, K]^T,
//   K = taps x input channels, walked in K=16 steps (two 8-channel "units" per step).
// Precision: the reference computes in fp32.  A single fp16/tf32 pass misses the 1e-3 parity bar
// (measured 1.2e-3..2.7e-3, DESIGN.md §precision), so every operand is an fp16 pair x = hi + lo and each
// K step issues three MMAs  hi*hi + lo*hi + hi*lo  (fp32 accumulation): ~2^-21 relative error while |x| >= 2^-3, which the
// weights get from a power-of-two prescale undone in the epilogue (ConvJob::w_unscale, DESIGN.md §2).
// The opt-in single pass (ConvJob::single, fav_net_set_precision "fp16"; template flag PAIR == false) issues hi*hi alone and
// copies only the hi planes of the patch and of each weight chunk: fp16 operands, fp32 accumulation.
//
// Data movement: the input patch of a tile (all filter rows x a group of channel blocks x 128+halo pixels)
// is fetched ONCE per tile by 1-D bulk async copies (cp.async.bulk, completion on an mbarrier).  Because the
// operand layout in HBM is already the canonical no-swizzle K-major core-matrix layout (net_layout.cuh), every
// filter tap reuses the same shared-memory patch: the wgmma matrix descriptor just starts 16 B * dx further.
// Weights stream through a ring of pre-packed chunks (or stay resident when the layer's weights fit).
//
// Warp roles (persistent CTAs, 1 per SM):
//   warps 0-7   two consumer warpgroups: warpgroup w issues the wgmmas of tile pixels [64w, 64w + 64) (M = 64, N = Npad,
//               accumulators in registers) and runs their epilogue: +bias -> stores + fused InstanceNorm statistics
//               (or x-fold reduction + tanh/deprocess for the last layer)
//   warp  8     B producer (bulk copies of weight chunks)
//   warp  9     A producer (bulk copies of the patch, all lanes issue)
//   warps 9-15  norm-on-load jobs: patch producers (raw fp32 -> InstanceNorm + ReLU -> fp16 hi/lo staged for the MMA,
//               replacing a separate in_apply pass)
// Plans per layer family (conv_plan.hpp): generic, stride-2 parity split, tap pairing (Cin = 8), x-fold; the sub-pixel phases
// of a stride-2 transposed conv stacked along N (plan_phase_stack).
// Pipelines: A stages and weight slots with full/empty mbarriers; each consumer warpgroup releases a slot once its
// wgmmas that read it have completed.
#include <atomic>

#include "conv.cuh"
#include "tc_common.cuh"
#include "wgmma_f16.cuh"

namespace fav {

constexpr int kMaxA = 4;  // patch stages
constexpr int kMaxB = 16;  // weight slots (ring or resident)
constexpr int kConsumerThreads = 256;  // warps 0-7
constexpr int kBWarp = 8, kAWarp = 9;
// norm-on-load producers: warps 9..15.  Seven warps fill the 512 threads one CTA can have at the 128 registers the consumers
// need; the producers are latency bound (one L2 round trip per unit of work), so each warp more adds loads in flight
constexpr int kNlWarps = 7;
constexpr int kThreads = kConsumerThreads + 32 * (1 + kNlWarps);  // launched with 320 threads when nl == 0
constexpr int kNlPx = 5;        // pixels in flight per lane (5 x 32 >= the 130-pixel patch row)
constexpr int kNlMaxC = 256;
constexpr int kExchPitch = 33;  // fp32 words per pixel in the x-fold exchange buffer (odd: conflict-free)
constexpr uint64_t kDescHi = (uint64_t)8u << 32;  // matrix descriptor: SBO = 8 x 16 B between 8-row core-matrix groups

struct __align__(16) TcShared {
  uint64_t a_full[kMaxA], a_empty[kMaxA], b_full[kMaxB], b_empty[kMaxB];
};

__device__ __forceinline__ float tc_final_value(float v, int k, int mode, float tanh_c) {
  float t = tanhf(v) * tanh_c;  // nn.Tanh -> nn.MulConstant(150) (models_video.lua:135-136)
  if (mode == 2) {              // fused vgg.deprocess (preprocess.lua:70)
    const float mean[3] = {FAV_MEAN_B, FAV_MEAN_G, FAV_MEAN_R};
    t = __fdiv_rn(__fadd_rn(t, mean[k]), 255.0f);
  }
  return t;
}

// ---- optional per-CTA timeline (job.trace != null; tools/trace_conv.py) ------------------------------------------------
// word 0: globaltimer at entry (ns), 1: clock64 at entry, 2: clock64 after setup, 3: clock64 at exit, 4: units of this CTA.
__device__ __forceinline__ void trace_put(const ConvJob &job, int word, long long v) {
  if (job.trace) job.trace[(size_t)blockIdx.x * kTraceWords + word] = (unsigned long long)v;
}

// fused statistics of image b: the 8 warps' partial sums of each accumulator column added in a FIXED order (deterministic per
// CTA: the tile -> CTA assignment is static), then one double atomic per column and quantity per CTA into its channel
// (stats_channel: a stacked job's phases add into the same channels one after the other).  reset: the partials are zeroed for
// the next image (thread ch clears the column it has just read; the closing barrier keeps the next tile's writers behind it).
__device__ __forceinline__ void tc_flush_stats(const ConvJob &job, float *slot, int b, bool reset) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  const int ch = threadIdx.x;  // accumulator column
  if (ch < stats_columns(job)) {
    float ssum = 0.f, qsum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) { ssum += slot[w * 256 + ch]; qsum += slot[w * 256 + 128 + ch]; }
    double *st = job.stats + b * job.stats_img;
    const int c = stats_channel(job, ch);
    atomicAdd(st + c, (double)ssum);
    atomicAdd(st + job.stats_pitch + c, (double)qsum);
  }
  if (reset) {
    if (ch < 128)
#pragma unroll
      for (int w = 0; w < 8; ++w) { slot[w * 256 + ch] = 0.f; slot[w * 256 + 128 + ch] = 0.f; }
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
}

// fused statistics of one column pair: v = {pixel r0: c, c + 1, pixel r0 + 8: c, c + 1} (zero where not stored) summed over the
// warp's 16 pixels (the 8 lanes that share lane % 4), then added into the warp's slot of accumulator columns c, c + 1 by one
// writer per (warp, column): deterministic
__device__ __forceinline__ void tc_stats_add(float *slot, int warp, int lane, int c, const float v[4]) {
  float s0 = v[0] + v[2], s1 = v[1] + v[3], t0 = v[0] * v[0] + v[2] * v[2], t1 = v[1] * v[1] + v[3] * v[3];
#pragma unroll
  for (int m = 4; m < 32; m <<= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, m); s1 += __shfl_xor_sync(0xffffffffu, s1, m);
    t0 += __shfl_xor_sync(0xffffffffu, t0, m); t1 += __shfl_xor_sync(0xffffffffu, t1, m);
  }
  if (lane < 4) {
    float *sl = slot + warp * 256;
    sl[c] += s0; sl[c + 1] += s1; sl[128 + c] += t0; sl[128 + c + 1] += t1;
  }
}

// consumer warpgroup: MMAs of one 64-pixel half of every tile of this CTA, then its epilogue.
// OPND: operand epilogue of batch-normalized nets (ConvJob::opnd) -- a template parameter, so the raw-output instances keep
// their code and registers.  BATCH: nimg > 1.  The same code; BATCH == false compiles it with nimg == 1 (one image, every
// image offset zero), so a single-frame launch keeps the code of a kernel without batches (about 1.5 % of a 720p frame).
// PAIR: the fp16 pair's three MMAs per K step; false: the single pass (ConvJob::single), hi * hi only.
template <int NT, bool OPND, bool BATCH, bool PAIR>
__device__ __forceinline__ void tc_consume(const ConvJob &job, uint8_t *a_base, uint8_t *b_base, TcShared *sh, float *exch) {
  constexpr int NJ = NT / 8;
  const int wg = threadIdx.x >> 7, wt = threadIdx.x & 127, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t a_stage_bytes = (uint32_t)job.stage16 * 16u, chunk_bytes = (uint32_t)job.chunk16 * 16u;
  const uint32_t nstages = (uint32_t)job.a_stages, nslots = (uint32_t)job.b_slots;
  const int ngroups = job.ngroups, nchunks = job.nchunks, spc = job.spc;
  const uint32_t b_step16 = 2u * (uint32_t)NT, b_lo16 = (uint32_t)spc * b_step16, a_stage16 = (uint32_t)job.stage16;
  const uint32_t *steps32 = reinterpret_cast<const uint32_t *>(job.steps);
  // this thread's accumulator rows (pixels of the tile) and column pairs
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), q2 = 2 * (lane & 3);
  float *slot = exch + 256;  // fused statistics: per-warp partial sums [8 warps][2][128], fixed summation order
  float acc[NT / 2];
  uint32_t sa = 0, aph = 0, sb = 0, bph = 0, tl = 0;
  const int total = (BATCH ? job.nimg : 1) * job.ntiles;
  for (int tile = blockIdx.x; tile < total;) {
    // this CTA's tiles of one image (tile_at), then that image's fused statistics: a CTA's tiles can cross into the next image, so
    // the slot partials go out (and are cleared) before the next image's tiles add to them -- each image gets the per-CTA sums it
    // gets when it runs alone (DESIGN.md 4.1)
    const TileAt img = tile_at(job, tile, BATCH);
    const int img_end = min(total, (img.b + 1) * job.ntiles);
    // the bias and scales of this image's style (style_at): the images of a batch may run different weight sets.  A single
    // image reads the job's own (written out at each use, which keeps the code of those instances as it was)
    StyleAt sty{};
    if constexpr (BATCH) sty = style_at(job, img.b);
    for (; tile < img_end; tile += gridDim.x, ++tl) {
      if (job.b_resident) sb = 0;
      uint32_t scale = 0;
      // one chunk of wgmmas stays in flight while the next is issued: a weight slot is released once the following chunk
      // is committed and the slot's own chunk has completed, a patch stage once the last chunk that read it has completed
      uint32_t b_prev = 0, a_prev = 0;
      for (int g = 0; g < ngroups; ++g) {
        mbar_wait(&sh->a_full[sa], aph);
        // A descriptor start: pixel r of the patch is at +16 B * r, this warpgroup's rows begin 64 pixels in
        const uint32_t a_hi16 = (smem_u32(a_base + sa * 2 * a_stage_bytes) >> 4) + (uint32_t)wg * 64u, a_lo16 = a_hi16 + a_stage16;
        uint32_t sidx = 0;
        for (int c = 0; c < nchunks; ++c) {
          if (!job.b_resident || tl == 0) mbar_wait(&sh->b_full[sb], job.b_resident ? 0u : bph);
          const uint32_t bh = (smem_u32(b_base + sb * chunk_bytes) >> 4) | ((uint32_t)NT << 16);  // LBO = Npad rows
          wgmma_fence();
          uint32_t bs = bh;
          for (int st = 0; st < spc; ++st, bs += b_step16) {
            const uint32_t dls = steps32[sidx + st];  // a_off16 | lbo16 << 16 (conv.cuh KStep)
            const uint64_t ad_hi = kDescHi | (a_hi16 + dls), ad_lo = kDescHi | (a_lo16 + dls);
            const uint64_t bd_hi = kDescHi | bs, bd_lo = kDescHi | (bs + b_lo16);
            Wgmma<NT>::mma(acc, ad_hi, bd_hi, scale);
            if constexpr (PAIR) {
              Wgmma<NT>::mma(acc, ad_lo, bd_hi, 1u);
              Wgmma<NT>::mma(acc, ad_hi, bd_lo, 1u);
            }
            scale = 1;
          }
          wgmma_commit();
          wgmma_wait<1>();  // every chunk but this one has completed
          if ((g | c) && wt == 0) {
            if (!job.b_resident) mbar_arrive(&sh->b_empty[b_prev]);
            if (c == 0) mbar_arrive(&sh->a_empty[a_prev]);
          }
          b_prev = sb;
          sidx += (uint32_t)spc;
          if (++sb == nslots) { sb = 0; bph ^= 1; }
        }
        a_prev = sa;
        if (++sa == nstages) { sa = 0; aph ^= 1; }
      }
      wgmma_wait<0>();
      if (wt == 0) {
        if (!job.b_resident) mbar_arrive(&sh->b_empty[b_prev]);
        mbar_arrive(&sh->a_empty[a_prev]);
      }
      if (job.dbg & 8) continue;

      // ===== epilogue from registers: acc[4i + 2h + e] = (pixel r0 + 8h, column 8i + q2 + e), in units of the weights times
      // 2^w_exp: every store takes acc * 2^-w_exp (exact) before the bias =====
      const TileAt at = tile_at(job, tile, BATCH);  // y, x0; the image's offsets are img's
      const int x0 = at.x0, y = at.y, yo = y * job.oy_mul + job.oy_off;
      const float ws = OPND ? 1.f : (BATCH ? sty.w_unscale : job.w_unscale);  // the operand epilogue's epi_scale includes it
      if (job.xfold_kw) {
        // partial sums Q[pixel][kx*Cout + co] -> shared memory, then out[x][co] = sum_kx Q[x + kx][kx*Cout + co]
        const int ncol = job.xfold_kw * job.Cout;
  #pragma unroll
        for (int i = 0; i < NJ; ++i)
  #pragma unroll
          for (int h = 0; h < 2; ++h)
  #pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * i + q2 + e;
              if (col < ncol) exch[(r0 + 8 * h) * kExchPitch + col] = acc[4 * i + 2 * h + e] * ws;
            }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int px = threadIdx.x, x = x0 + px;
        if (px < job.tile_dx && x < job.Wo && y < job.Ho && !(job.dbg & 1)) {
          const int xo = x * job.ox_mul + job.ox_off;
          const float *qv = exch + px * kExchPitch;
          const int64_t plane = (int64_t)job.Ho * job.Wo, o = (int64_t)yo * job.Wo + xo;
          for (int k = 0; k < job.Cout; ++k) {
            float sum = __ldg((BATCH ? sty.bias : job.bias) + k);
            for (int kx = 0; kx < job.xfold_kw; ++kx) sum += qv[kx * (kExchPitch + job.Cout) + k];
            job.out3[img.out3 + (job.final_mode == 2 ? 2 - k : k) * plane + o] = tc_final_value(sum, k, job.final_mode, job.tanh_c);
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");  // exch is rewritten by the next tile
        continue;
      }
      bool valid[2];
      int xo[2];
  #pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int x = x0 + r0 + 8 * h;
        valid[h] = x < job.Wo && y < job.Ho && !(job.dbg & 1);
        xo[h] = x * job.ox_mul + job.ox_off;
      }
      if (job.final_mode) {
        // Cout <= 3 output channels sit in column group 0
  #pragma unroll
        for (int h = 0; h < 2; ++h)
  #pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = q2 + e;
            if (k < 3 && k < job.Cout && valid[h])
              job.out3[img.out3 + ((int64_t)(job.final_mode == 2 ? 2 - k : k) * job.Ho + yo) * job.Wo + xo[h]] =
                  tc_final_value(fmaf(acc[2 * h + e], ws, __ldg((BATCH ? sty.bias : job.bias) + k)), k, job.final_mode, job.tanh_c);
          }
        continue;
      }
      if (!OPND && job.nstack) {
        // stacked sub-pixel phases: column pair n of phase s = n / Cout goes to that phase's output pixel (stack_epi_addr); its
        // statistics stay in column n until tc_flush_stats
        const bool stats = job.stats && !(job.dbg & 64);
        float *raw = job.raw + img.raw;
  #pragma unroll
        for (int i = 0; i < NJ; ++i) {
          const int n = 8 * i + q2;
          const float2 b = __ldg(reinterpret_cast<const float2 *>((BATCH ? sty.bias : job.bias) + n));  // the bias of each stacked phase
          float v[4];
  #pragma unroll
          for (int h = 0; h < 2; ++h) {
            int64_t o = 0;
            v[2 * h] = fmaf(acc[4 * i + 2 * h], ws, b.x);
            v[2 * h + 1] = fmaf(acc[4 * i + 2 * h + 1], ws, b.y);
            if (stack_epi_addr(job, y, x0, threadIdx.x, i, h, o) && !(job.dbg & 1))
              *reinterpret_cast<float2 *>(raw + o) = make_float2(v[2 * h], v[2 * h + 1]);
            else
              v[2 * h] = v[2 * h + 1] = 0.f;
          }
          if (stats) tc_stats_add(slot, warp, lane, n, v);
        }
        continue;
      }
      if constexpr (OPND) {
        // the two channels c, c + 1 of each of the thread's two pixels: BN scale and bias (+ReLU) (+skip) -> fp16 hi / lo pair, one 4-byte store
        // per plane; the 4 lanes of a quad fill one 16-byte (pixel, channel block) cell.  No statistics, no atomics.
        uint32_t *dhi = reinterpret_cast<uint32_t *>(job.epi_dst.hi), *dlo = reinterpret_cast<uint32_t *>(job.epi_dst.lo);
  #pragma unroll
        for (int i = 0; i < NJ; ++i) {
          const int c = 8 * i + q2;
          // bias and scale are padded to Npad; the scale includes the weights' 2^-w_exp (pack_conv_weights, net.cu)
          const float2 b = __ldg(reinterpret_cast<const float2 *>((BATCH ? sty.bias : job.bias) + c)),
                     s = __ldg(reinterpret_cast<const float2 *>((BATCH ? sty.epi_scale : job.epi_scale) + c));
  #pragma unroll
          for (int h = 0; h < 2; ++h) {
            int64_t o, so;
            // (a single image decodes the tile per store, as the register allocation of the unbatched kernel prefers)
            if (!(BATCH ? opnd_epi_addr(job, at, threadIdx.x, i, h, o, so) : opnd_epi_addr(job, tile, threadIdx.x, i, h, o, so, false)))
              continue;
            float v0 = fmaf(acc[4 * i + 2 * h], s.x, b.x), v1 = fmaf(acc[4 * i + 2 * h + 1], s.y, b.y);
            if (job.epi_relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (job.epi_skip) {  // ConcatTable{conv_block, ShaveImage / Identity} -> CAddTable; same arithmetic as in_apply
              const uint32_t sh = __ldg(reinterpret_cast<const uint32_t *>(job.epi_skip_op.hi) + so);
              const uint32_t sl = __ldg(reinterpret_cast<const uint32_t *>(job.epi_skip_op.lo) + so);
              const float2 fh = __half22float2(*reinterpret_cast<const __half2 *>(&sh));
              const float2 fl = __half22float2(*reinterpret_cast<const __half2 *>(&sl));
              v0 += fh.x + fl.x; v1 += fh.y + fl.y;
            }
            uint32_t hw, lw;
            split_pair(v0, v1, hw, lw);
            dhi[o] = hw; dlo[o] = lw;
          }
        }
        continue;
      }
      const bool stats = job.stats && !(job.dbg & 64);
      float *raw = job.raw + img.raw;
  #pragma unroll
      for (int i = 0; i < NJ; ++i) {
        const int c = 8 * i + q2;
        const float2 b = __ldg(reinterpret_cast<const float2 *>((BATCH ? sty.bias : job.bias) + c));
        float v[4];
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[2 * h] = fmaf(acc[4 * i + 2 * h], ws, b.x);
          v[2 * h + 1] = fmaf(acc[4 * i + 2 * h + 1], ws, b.y);
          // raw layout [Ho][Cq][Wp][4]: channels c, c + 1 of one pixel are 8 contiguous bytes
          if (valid[h] && c < job.Cout)
            *reinterpret_cast<float2 *>(raw + (((int64_t)yo * job.raw_Cq + (c >> 2)) * job.raw_Wp + xo[h]) * 4 + (c & 3)) =
                make_float2(v[2 * h], v[2 * h + 1]);
          if (!valid[h]) v[2 * h] = v[2 * h + 1] = 0.f;
        }
        if (stats) tc_stats_add(slot, warp, lane, c, v);
      }
    }
    if (!OPND && job.stats) tc_flush_stats(job, slot, img.b, tile < total);  // an operand epilogue has no statistics
  }
}

// norm-on-load table of image b (threads tid, tid + nthr, ...), with the gamma / beta of its style (style_at)
template <bool BATCH>
__device__ __forceinline__ void nl_build_table(const ConvJob &job, float *nl_tab, int b, int tid, int nthr) {
  const double *sums = job.nl_sums + b * job.nl_sums_img;
  const float *gamma = job.nl_gamma, *beta = job.nl_beta;
  if constexpr (BATCH) {
    const StyleAt sty = style_at(job, b);
    gamma = sty.nl_gamma; beta = sty.nl_beta;
  }
#pragma unroll 1  // kept rolled: an unrolled copy inside the producer loop costs the OPND instances a 4-byte spill
  for (int c = tid; c < job.nl_C; c += nthr) {
    in_finalize(sums[c], sums[job.nl_C + c], job.nl_inv_count, job.nl_eps, gamma[c], nl_tab[c], nl_tab[kNlMaxC + c]);
    nl_tab[2 * kNlMaxC + c] = beta[c];
  }
}

template <int NT, bool OPND, bool BATCH, bool PAIR>
__global__ void __launch_bounds__(kThreads, 1) conv_tc_kernel(const __grid_constant__ ConvJob job) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t a_stage_bytes = (uint32_t)job.stage16 * 16u;  // one of hi / lo
  const uint32_t chunk_bytes = (uint32_t)job.chunk16 * 16u;
  uint8_t *a_base = smem;                                   // stage s: hi | lo
  const uint32_t nstages = (uint32_t)job.a_stages;
  uint8_t *b_base = a_base + nstages * 2 * a_stage_bytes;   // slot s: [hi steps][lo steps]
  const uint32_t nslots = (uint32_t)job.b_slots;
  TcShared *sh = reinterpret_cast<TcShared *>(b_base + nslots * chunk_bytes);
  float *exch = reinterpret_cast<float *>(sh + 1);  // x-fold exchange buffer [128][kExchPitch] / statistics slots

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (job.trace && threadIdx.x == 0) {
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    trace_put(job, 0, (long long)gt);
    trace_put(job, 1, clock64());
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < kMaxA; ++i) { mbar_init(&sh->a_full[i], job.nl ? kNlWarps : 1); mbar_init(&sh->a_empty[i], 2); }
    for (int i = 0; i < kMaxB; ++i) { mbar_init(&sh->b_full[i], 1); mbar_init(&sh->b_empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (job.stats && !job.xfold_kw)
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) exch[256 + i] = 0.f;
  // norm-on-load: mean / gamma*rstd / beta per input channel from the producer conv's fused statistics (same arithmetic
  // as in_apply_kernel: biased variance, eps inside the sqrt, InstanceNormalization.lua:39-50)
  // (after the x-fold exchange buffer, or after the statistics slots: tc_fixed_smem)
  float *nl_tab = exch + (job.xfold_kw ? kTileM * kExchPitch : 256 + 8 * 2 * 128);
  const int total = (BATCH ? job.nimg : 1) * job.ntiles;
  int nl_b = BATCH ? (int)blockIdx.x / job.ntiles : 0;  // image whose statistics nl_tab holds
  if (job.nl) nl_build_table<BATCH>(job, nl_tab, nl_b, threadIdx.x, blockDim.x);
  __syncthreads();
  if (threadIdx.x == 0 && job.trace) trace_put(job, 2, clock64());

  const int ngroups = job.ngroups, nchunks = job.nchunks;

  if (warp < 8) {
    tc_consume<NT, OPND, BATCH, PAIR>(job, a_base, b_base, sh, exch);
  } else if (job.nl && warp >= kAWarp) {
    // ===== norm-on-load patch producers: raw fp32 -> InstanceNorm (+ReLU) -> fp16 hi/lo -> MMA-ready stage (hi only: !PAIR) =====
    // The warps take turns over units of 32 kNlPx pixels of one (patch row, channel block) slab: lanes run along the slab,
    // kNlPx float4 pairs in flight per lane.  Units rather than whole slabs keep the warps evenly loaded when a slab is longer
    // than one unit (the 257 pixels of a stride-2 consumer).
    const int pw = warp - kAWarp;
    const int pslab = job.pslab16, nck = (pslab + 32 * kNlPx - 1) / (32 * kNlPx), nunits = job.nrows * job.CbG * nck;
    uint32_t s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const TileAt at = tile_at(job, tile, BATCH);
      const int y = at.y, x0 = at.x0;
      if (at.b != nl_b) {
        // the next image (and its style): its table replaces the current one once all producer warps are done with the
        // previous tile
        nl_b = at.b;
        asm volatile("bar.sync 2, %0;" ::"r"(32 * kNlWarps) : "memory");
        nl_build_table<BATCH>(job, nl_tab, nl_b, threadIdx.x - kAWarp * 32, 32 * kNlWarps);
        asm volatile("bar.sync 2, %0;" ::"r"(32 * kNlWarps) : "memory");
      }
      const float4 *nl_raw = job.nl_raw + at.nl_raw4;
      for (int g = 0; g < ngroups; ++g) {
        mbar_wait(&sh->a_empty[s], ph ^ 1);
        uint8_t *stage = a_base + s * 2 * a_stage_bytes;
        for (int u = pw; u < nunits; u += kNlWarps) {
          const int rc = u / nck, pb = (u - rc * nck) * 32 * kNlPx;
          const int ri = rc / job.CbG, cbi = rc - ri * job.CbG;
          const int ry = nl_raw_row(job, y, g, ri), cb = job.grp_cb0[g] + cbi;
          const bool row_ok = ry >= 0 && ry < job.nl_H;
          const float4 *rp = nl_raw + ((int64_t)(row_ok ? ry : 0) * job.nl_Cq + 2 * cb) * job.nl_Wp;
          float tm[8], ts[8], tb[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) { tm[i] = nl_tab[cb * 8 + i]; ts[i] = nl_tab[kNlMaxC + cb * 8 + i]; tb[i] = nl_tab[2 * kNlMaxC + cb * 8 + i]; }
          uint8_t *drow = stage + (uint32_t)(rc * pslab) * 16u;
          {
            float4 va[kNlPx], vb[kNlPx];
            uint32_t okm = 0;
#pragma unroll
            for (int k = 0; k < kNlPx; ++k) {
              const int p = pb + k * 32 + lane, x = nl_raw_col(job, x0, p);
              const bool ok = row_ok && p < pslab && x >= 0 && x < job.nl_W;
              // unconditional loads from a clamped (always valid) address: all 2 * kNlPx requests are issued back to back
              const int xc = x < 0 ? 0 : (x < job.nl_Wp ? x : job.nl_Wp - 1);
              va[k] = __ldg(rp + xc); vb[k] = __ldg(rp + job.nl_Wp + xc);
              if (ok) okm |= 1u << k;
            }
#pragma unroll
            for (int k = 0; k < kNlPx; ++k) {
              const int p = pb + k * 32 + lane;
              if (p >= pslab) continue;
              float v[8] = {va[k].x, va[k].y, va[k].z, va[k].w, vb[k].x, vb[k].y, vb[k].z, vb[k].w};
              if (!(okm & (1u << k))) {  // pixels outside the image are zero (never normalised)
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = 0.f;
              } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  const float t = (v[i] - tm[i]) * ts[i] + tb[i];
                  v[i] = job.nl_relu ? fmaxf(t, 0.f) : t;
                }
              }
              uint32_t h[4], l[4];  // same values as split_store8 (net_kernels.cu), packed two per conversion
#pragma unroll
              for (int i = 0; i < 4; ++i) split_pair(v[2 * i], v[2 * i + 1], h[i], l[i]);
              *reinterpret_cast<uint4 *>(drow + (uint32_t)p * 16u) = make_uint4(h[0], h[1], h[2], h[3]);
              if constexpr (PAIR)
                *reinterpret_cast<uint4 *>(drow + a_stage_bytes + (uint32_t)p * 16u) = make_uint4(l[0], l[1], l[2], l[3]);
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to wgmma
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh->a_full[s]);
        if (++s == nstages) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp == kAWarp) {
    // ===== A producer: the input patch of each (tile, channel group): one bulk copy per (patch row, channel block, hi/lo),
    // spread over the 32 lanes (hi only: !PAIR) =====
    constexpr int NP = PAIR ? 2 : 1;              // planes copied
    const int per_row = job.CbG * job.nseg * NP;  // copies per patch row
    const int ncopies = job.nrows * per_row;
    const uint32_t stage_tx = tc_a_stage_tx(job, PAIR);
    uint32_t s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const TileAt at = tile_at(job, tile, BATCH);
      const int y = at.y, x0 = at.x0;
      for (int g = 0; g < ngroups; ++g) {
        mbar_wait(&sh->a_empty[s], ph ^ 1);
        if (lane == 0) mbar_arrive_expect_tx(&sh->a_full[s], stage_tx);
        __syncwarp();
        uint8_t *stage = a_base + s * 2 * a_stage_bytes;
        for (int c = lane; c < ncopies; c += 32) {
          int ri = c / per_row, r = c - ri * per_row;
          int cbi = r / (job.nseg * NP);
          r -= cbi * job.nseg * NP;
          int seg = PAIR ? r >> 1 : r, part = PAIR ? r & 1 : 0;
          int64_t src16 = ((int64_t)(job.row_mul * y + job.grp_row[g][ri]) * job.a_Cb + job.grp_cb0[g] + cbi) *
                              job.a_slab16 + job.seg_src16[seg] + x0 + at.a16;
          const uint4 *src = (part ? job.a_lo : job.a_hi) + src16;
          uint8_t *dst = stage + part * a_stage_bytes +
                         (uint32_t)((ri * job.CbG + cbi) * job.pslab16 + job.seg_dst16[seg]) * 16u;
          bulk_g2s(dst, src, (job.dbg & 4) ? 16u : (uint32_t)job.seg_len16[seg] * 16u, &sh->a_full[s]);
        }
        if (++s == nstages) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp == kBWarp) {
    // ===== B producer: weight chunks (the hi steps, the first half of each chunk, only: !PAIR), from the style of the tile's
    // image (style_at; a net with several styles streams every job's weights, conv_tc_choose_slots) =====
    if (lane == 0) {
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        if (job.b_resident && tile != (int)blockIdx.x) break;  // resident weights: one pass fills every slot
        const uint4 *wb = BATCH ? style_at(job, tile_at(job, tile).b).b : job.b;
        for (int g = 0; g < ngroups; ++g)
          for (int c = 0; c < nchunks; ++c) {
            mbar_wait(&sh->b_empty[s], ph ^ 1);
            const uint32_t cb = FAV_TC_B_CHUNK_TX(job.dbg, chunk_bytes, PAIR);
            mbar_arrive_expect_tx(&sh->b_full[s], cb);
            bulk_g2s(b_base + s * chunk_bytes, wb + (int64_t)(g * nchunks + c) * job.chunk16, cb, &sh->b_full[s]);
            if (++s == nslots) { s = 0; ph ^= 1; }
          }
      }
    }
    __syncwarp();
  }

  __syncthreads();
  if (threadIdx.x == 0 && job.trace) {
    trace_put(job, 3, clock64());
    int nu = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) ++nu;
    trace_put(job, 4, nu);
  }
}

static size_t tc_fixed_smem(const ConvJob &job) {
  return (size_t)job.a_stages * 2 * job.stage16 * 16 + sizeof(TcShared) + 128 +
         (job.xfold_kw ? (size_t)kTileM * kExchPitch * 4 : job.opnd ? 0 : (size_t)(256 + 8 * 2 * 128) * 4) +
         (job.nl ? (size_t)3 * kNlMaxC * 4 : 0);
}
size_t conv_tc_smem_bytes(const ConvJob &job) { return tc_fixed_smem(job) + (size_t)job.b_slots * job.chunk16 * 16; }

void conv_tc_choose_slots(ConvJob &job) {
  const size_t budget = 224 * 1024, chunk = (size_t)job.chunk16 * 16;
  const int total = job.rf_R ? job.rf_steps : (job.pf ? job.ngroups * 4 : job.ngroups * job.nchunks);
  job.a_stages = 2;
  // small-work groups (resident weights, several groups per tile) are latency bound on the patch pipeline:
  // deepen it while everything still fits
  {
    ConvJob t = job;
    for (int n = kMaxA; n > 2; --n) {
      t.a_stages = n;
      if (total <= kMaxB && tc_fixed_smem(t) + total * chunk <= budget) { job.a_stages = n; break; }
    }
  }
  if (const char *e = getenv("FAV_ASTAGES")) {  // tuning knob: force the patch ring depth (weights take what is left)
    const int n = atoi(e);
    ConvJob t = job;
    t.a_stages = n;
    if (n >= 2 && n <= kMaxA && tc_fixed_smem(t) + 2 * chunk <= budget) job.a_stages = n;
  }
  const size_t fixed = tc_fixed_smem(job);
  // a banked job streams its chunks through the ring, per tile from the tile's style (tc_may_keep_weights)
  if (total <= kMaxB && fixed + total * chunk <= budget && tc_may_keep_weights(job)) {
    job.b_resident = 1;
    job.b_slots = total;
  } else {
    job.b_resident = 0;
    int n = (int)((budget - fixed) / chunk);
    job.b_slots = n > kMaxB ? kMaxB : (n < 2 ? 2 : n);
  }
}

// diagnostics: device buffer receiving the timeline of the next launches (kTraceWords u64 per CTA, launches appended)
static unsigned long long *g_trace_buf = nullptr;
static size_t g_trace_cap = 0, g_trace_used = 0;
void conv_tc_set_trace(unsigned long long *buf, size_t words) { g_trace_buf = buf; g_trace_cap = words; g_trace_used = 0; }
size_t conv_tc_trace_used() { return g_trace_used; }
unsigned long long *conv_trace_claim(size_t words) {
  if (!g_trace_buf || g_trace_used + words > g_trace_cap) return nullptr;
  unsigned long long *p = g_trace_buf + g_trace_used;
  g_trace_used += words;
  return p;
}

int launch_conv_tc(const ConvJob &job_in, int num_sms, cudaStream_t st) {
  ConvJob job = job_in;
  if (job.mt != 1 || job.rf_R || job.pf || job.ksplit) {
    set_error("conv_tc: plan with mt=%d rf_R=%d pf=%d ksplit=%d has no wgmma kernel", job.mt, job.rf_R, job.pf, job.ksplit);
    return FAV_ERR_UNSUPPORTED;
  }
  void (*kernel)(ConvJob) = nullptr;
  // a job with a style table runs the batched instances for one image too: they look the image's style up (style_at)
  const bool batch = job.nimg > 1 || job.img_style, pair = !job.single;
#define FAV_TC_PICK(N, P)                                                                                      \
  (job.opnd ? (batch ? conv_tc_kernel<N, true, true, P> : conv_tc_kernel<N, true, false, P>)                   \
            : (batch ? conv_tc_kernel<N, false, true, P> : conv_tc_kernel<N, false, false, P>))
#define FAV_TC_CASE(N)                                                                                         \
  case N:                                                                                                      \
    kernel = pair ? FAV_TC_PICK(N, true) : FAV_TC_PICK(N, false);                                              \
    break;
  switch (job.Npad) {
    FAV_TC_CASE(16) FAV_TC_CASE(32) FAV_TC_CASE(48) FAV_TC_CASE(64) FAV_TC_CASE(80) FAV_TC_CASE(96) FAV_TC_CASE(112)
    FAV_TC_CASE(128)
    default:
      set_error("conv_tc: no wgmma kernel for N = %d (multiples of 16 up to 128)", job.Npad);
      return FAV_ERR_UNSUPPORTED;
  }
#undef FAV_TC_CASE
#undef FAV_TC_PICK
  // one persistent CTA per SM over the tiles of every image (tile_at); the grid of a single image is unchanged
  const int total = job.nimg * job.ntiles, grid = total < num_sms ? total : num_sms;
  job.trace = conv_trace_claim((size_t)grid * kTraceWords);
  size_t smem = conv_tc_smem_bytes(job);
  if (smem > 227 * 1024) {
    set_error("conv_tc: shared memory %zu exceeds 227 KB", smem);
    return FAV_ERR_UNSUPPORTED;
  }
  // the opt-in to > 48 KB of dynamic shared memory is a PER-DEVICE attribute of each instantiation
  static std::atomic<uint64_t> attr_set[72];
  int dev = 0;
  FAV_TRY(check_cuda(cudaGetDevice(&dev), "cudaGetDevice"));
  const uint64_t bit = 1ull << (dev & 63);
  std::atomic<uint64_t> &set = attr_set[job.Npad / 16 + (job.opnd ? 9 : 0) + (batch ? 18 : 0) + (pair ? 0 : 36)];
  if (!(set.load(std::memory_order_acquire) & bit)) {
    FAV_TRY(check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024),
                       "cudaFuncSetAttribute(conv_tc)"));
    set.fetch_or(bit, std::memory_order_release);
  }
  kernel<<<grid, job.nl ? kThreads : kConsumerThreads + 64, smem, st>>>(job);
  return post_launch("conv_tc");
}

}  // namespace fav

extern "C" {
// diagnostics: timeline of the following conv_tc launches into a caller-owned device buffer (bytes / 8 u64 words);
// NULL switches it off.  Used by tools/trace_conv.py through fav_net_forward (graph launches keep the pointer they captured).
int fav_debug_set_trace(void *dev_buf, size_t bytes) {
  fav::conv_tc_set_trace(reinterpret_cast<unsigned long long *>(dev_buf), dev_buf ? bytes / 8 : 0);
  return FAV_OK;
}
size_t fav_debug_trace_words(void) { return fav::conv_tc_trace_used(); }
}
