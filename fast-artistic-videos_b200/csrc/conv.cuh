// conv.cuh -- job descriptors shared by the host planner (net.cu) and the convolution kernels.
#pragma once
#include "net_layout.cuh"

namespace fav {

constexpr int kMaxTaps = 81;
constexpr int kMaxSteps = 168;
constexpr int kMaxRfRows = 24;  // row-fold: R + KH - 1 patch rows per unit
constexpr int kMaxRows = 10;
constexpr int kMaxGroups = 12;
constexpr int kTileM = 128;  // output pixels per tile (two 64-row wgmma halves)
constexpr int kTraceWords = 64;   // u64 words per CTA in the optional timeline buffer
constexpr int kTraceUnits = 6;    // units (tiles) per CTA recorded

// One K=16 step of the implicit GEMM: two K8 "units" (a unit = 8 input channels of one filter tap).
// a_off16: offset (16-byte units) of the first unit's pixel 0 inside the shared-memory patch stage;
// lbo16:   distance between the two units (= patch slab pitch when they are adjacent channel blocks,
//          1 when they are horizontally adjacent taps of an 8-channel input).
struct KStep {
  uint16_t a_off16;
  uint16_t lbo16;
};

// tensor-core (wgmma) implicit-GEMM job (one convolution, or one sub-pixel phase of a transposed convolution)
struct ConvJob {
  // input operand (hi/lo fp16 planes), addressed in 16-byte units
  const uint4 *a_hi, *a_lo;
  int a_Cb, a_slab16;
  // output grid of this job and its tiling (one tile = 128 consecutive pixels of one output row)
  int Ho, Wo, tiles_x, ntiles;
  // patch geometry: storage row of patch row ri in group g for output row y: row_mul*y + grp_row[g][ri]
  int row_mul;
  int nseg, seg_src16[2], seg_len16[2], seg_dst16[2];  // bulk-copy segments per (row, cb): src + x0
  int ngroups, nrows, CbG;
  int grp_cb0[kMaxGroups];
  int grp_row[kMaxGroups][kMaxRows];
  int pslab16;   // patch slab pitch (16-byte units) per (row, cb)
  int stage16;   // one A stage (hi or lo) in 16-byte units
  int nchunks, spc;  // weight chunks per group, K16 steps per chunk
  KStep steps[kMaxSteps + 8];  // +spare: the issue loop reads kMaxSpc entries per chunk
  const uint4 *b;  // packed weights: [group][chunk][hi|lo][step][k8 half][Npad] x 16 B
  int chunk16;     // 2 * spc * 2 * Npad
  int Npad, Cout;
  const float *bias;
  // x-fold (final 9x9, Cout <= 4): the filter COLUMNS are folded into N (n = kx*Cout + co), the patch has no
  // horizontal halo, tiles advance by tile_dx = 128 - (KW-1) pixels and the epilogue adds the KW shifted partial
  // sums through a shared-memory exchange buffer.  xfold_kw == 0: plain mode, tile_dx == 128.
  int tile_dx, xfold_kw;
  // weight pipeline: b_slots ring slots of chunk16*16 bytes; b_resident: every chunk of the job has its own slot,
  // is loaded once per CTA and never released (small layers: no per-tile weight traffic)
  int b_slots, b_resident;
  int a_stages;  // patch pipeline depth (2..4), chosen from the shared-memory budget
  // mt: output rows per work unit (1 or 2).  mt = 2 shares every weight chunk and the overlapping patch rows between
  // two vertically adjacent 128-pixel tiles (M = 256, two accumulators): halves the weight traffic per pixel.
  int mt;
  // row-fold (tall filters with a narrow N block: conv1 9x9 7->32, x-folded final 9x9): a unit is rf_R output rows;
  // the patch is walked row by row and the MMA of patch row iy accumulates into ALL output rows r with
  // 0 <= iy - r < rf_kh at once: the resident weights are stored with the filter rows in DESCENDING ky order along N
  // (n = (rf_kh-1-ky)*rf_nblk + c), so the valid output rows of a patch row are a contiguous N-slice of the weights
  // and a contiguous column range of the accumulator.  3x fewer and fatter MMAs, patch re-read amplification
  // (rf_R + rf_kh - 1) / rf_R instead of rf_kh.  rf_R == 0: off.
  int rf_R, rf_kh, rf_nblk, rf_steps, rf_row16, rf_total_rows;
  // phase-fold (stride-2 transposed conv): the 4 sub-pixel phases are folded into N in the order
  // (a,b) = (0,0),(0,1),(1,1),(1,0) so that the phases fed by tap (dy,dx) are a contiguous block range:
  // tap(0,0) -> blocks 0..3, (0,1) -> 1..2, (1,0) -> 2..3, (1,1) -> 2.  One weight chunk per tap (pf_n = N of its MMAs,
  // pf_col = first accumulator column); the patch is loaded once for all phases and each thread stores 2x2 pixels.
  int pf;
  int pf_n[4], pf_col[4], pf_len16[4], pf_src16[4], pf_grp16, pf_cout;
  int ksplit;          // 1: two issuing warps take alternate K steps into two accumulators (columns +0 / +128)
  // row-fold: per patch row iy (host-computed, keeps the issue loop free of index arithmetic): accumulator column of
  // the first output row it feeds, weight-row offset of its slice, instruction descriptors for all / old / new rows
  uint32_t rf_dcol[kMaxRfRows], rf_boff[kMaxRfRows], rf_idn_all[kMaxRfRows], rf_idn_acc[kMaxRfRows], rf_idn_new[kMaxRfRows],
      rf_off_new[kMaxRfRows];
  // norm-on-load: the input is the RAW output of the previous convolution; InstanceNorm (+ReLU) and the fp16 hi/lo split
  // happen in the producer warps while the patch is staged (replaces a separate in_apply pass + operand round trip)
  int nl;
  const float4 *nl_raw; int nl_Cq, nl_Wp, nl_H, nl_W, nl_padT, nl_padL, nl_relu, nl_C;
  const double *nl_sums; const float *nl_gamma, *nl_beta; double nl_inv_count, nl_eps;
  // per-CTA timeline (diagnostics, fav_debug_set_trace): kTraceWords u64 per CTA, null = off.  Layout in conv_tc.cu.
  unsigned long long *trace;
  // timing ablations (env FAV_DBG, diagnostics only; results are wrong when non-zero): 1 = no epilogue stores/stats,
  // 2 = 16-byte weight copies, 4 = 16-byte patch copies, 8 = no epilogue at all
  int dbg;
  // fused InstanceNorm statistics: per-channel sum / sum of squares of the stored values (double, atomics), or null
  double *stats;
  // output placement: raw(y*oy_mul + oy_off, x*ox_mul + ox_off)
  float *raw;
  int raw_Cq, raw_Wp;
  int oy_mul, oy_off, ox_mul, ox_off;
  // final layer: Tanh -> MulConstant(tanh_c) [-> deprocess] written as fp32 NCHW [3][outH][outW]
  int final_mode;  // 0 = raw, 1 = net space, 2 = fused vgg.deprocess
  float *out3;
  float tanh_c;
};

// CUDA-core comparator job (debug / bring-up path; same inputs and outputs as ConvJob)
struct SimtJob {
  Operand in;
  int sy, sx;  // input stride
  int ntaps;
  int8_t tdy[kMaxTaps], tdx[kMaxTaps];
  const float *w;  // [tap][Cin_pad][Cout_pad8] fp32
  int Cin_pad, Cout, Cout_pad8;
  const float *bias;
  int Ho, Wo;
  float *raw;
  int raw_Cq, raw_Wp;
  int raw_planar, raw_Hp;  // planar raw output [C][Hp][Wp] (CUDA-core comparator only)
  int oy_mul, oy_off, ox_mul, ox_off;
  int final_mode;
  float *out3;
  float tanh_c;
};

int launch_conv_tc(const ConvJob &job, int num_sms, cudaStream_t st);
int launch_conv_simt(const SimtJob &job, cudaStream_t st);
size_t conv_tc_smem_bytes(const ConvJob &job);
void conv_tc_set_trace(unsigned long long *buf, size_t words);  // diagnostics (fav_debug_set_trace)
unsigned long long *conv_trace_claim(size_t words);             // next `words` u64 of the timeline buffer, or null
size_t conv_tc_trace_used();
void conv_tc_choose_slots(ConvJob &job);  // fills b_slots / b_resident from the shared-memory budget

// elementwise / reduction kernels of the net (net_kernels.cu)
int launch_pack_input(const float *in, int Cin, int H, int W, int reflect, const Operand &dst, cudaStream_t st);
int launch_in_stats(const RawTensor &raw, double *sums /*[2*C]*/, cudaStream_t st);
int launch_in_apply(const RawTensor &raw, const double *sums, const float *gamma, const float *beta, float eps, int relu,
                    const Operand *skip, int shave, const Operand &dst, cudaStream_t st);
int launch_up_in(const Operand &src, double *sums, const float *gamma, const float *beta, float eps, int relu, int scale,
                 const Operand &dst, cudaStream_t st);
int launch_unpack_operand(const Operand &src, float *out_nchw, cudaStream_t st);

}  // namespace fav
