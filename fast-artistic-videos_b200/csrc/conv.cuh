// conv.cuh -- job descriptors shared by the host planner (net.cu) and the convolution kernels.
#pragma once
#include "net_layout.cuh"

namespace fav {

constexpr int kMaxTaps = 81;
constexpr int kMaxSteps = 168;
constexpr int kMaxRfRows = 24;  // row-fold: R + KH - 1 patch rows per unit
constexpr int kMaxRows = 10;
constexpr int kMaxGroups = 16;  // K groups of one job: Cin = 512 in channel groups of 4 blocks (VGG-16 conv4_x)
constexpr int kMaxNBlock = 128;  // output channels of one job (wgmma N); wider convolutions run one job per N block
constexpr int kTileM = 128;  // output pixels per tile (two 64-row wgmma halves)
constexpr int kTraceWords = 64;   // u64 words per CTA in the optional timeline buffer
constexpr int kTraceUnits = 6;    // units (tiles) per CTA recorded

// The fp16 pair x = hi + lo carries ~22 significant bits only while lo is an fp16 normal, i.e. for |x| >= 2^-3 (lo's normals
// start at 2^-14).  A tensor packed multiplied by 2^pow2_scale_exp has its max |x| in [2^14, 2^15): clear of that floor and of
// the fp16 maximum 65504.  maxbits: the float bits of max |x|; 0 (an all-zero tensor) gives 0.  |e| <= 126 keeps 2^e and 2^-e
// normal.  The factor is exact, so it changes no rounding; whoever reads the fp32 result multiplies it by 2^-e.
__host__ __device__ inline int pow2_scale_exp(unsigned maxbits) {
  if (maxbits == 0) return 0;
  int e = (int)((maxbits >> 23) & 0xff);  // floor(log2 max) + 127; subnormals as 2^-126
  e = (e < 1 ? 1 : e) - 127;
  e = 14 - e;
  return e < -126 ? -126 : (e > 126 ? 126 : e);
}

// One K=16 step of the implicit GEMM: two K8 "units" (a unit = 8 input channels of one filter tap).
// a_off16: offset (16-byte units) of the first unit's pixel 0 inside the shared-memory patch stage;
// lbo16:   distance between the two units (= patch slab pitch when they are adjacent channel blocks,
//          1 when they are horizontally adjacent taps of an 8-channel input).
struct KStep {
  uint16_t a_off16;
  uint16_t lbo16;
};

// tensor-core (wgmma) implicit-GEMM job (one convolution, or one or several stacked sub-pixel phases of a transposed convolution)
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
  // fused InstanceNorm statistics: per-channel sum / sum of squares of the stored values (double, atomics), or null.
  // Channel c of this job adds into stats[c] and stats[stats_pitch + c]: stats_pitch is the whole tensor's channel count, so
  // the N blocks of a wide convolution fill disjoint slots of one [sum][sum of squares] array (conv_nblock_stats)
  double *stats;
  int stats_pitch;
  // output placement: raw(y*oy_mul + oy_off, x*ox_mul + ox_off)
  float *raw;
  int raw_Cq, raw_Wp;
  int oy_mul, oy_off, ox_mul, ox_off;
  // stacked sub-pixel phases of a stride-2 transposed conv (plan_phase_stack): accumulator column n = s * Cout + c is channel
  // c of phase s, placed at raw(y*oy_mul + st_oy[s], x*ox_mul + st_ox[s]) (stack_epi_addr).  0: one phase per job
  int nstack, st_oy[4], st_ox[4];
  // final layer: Tanh -> MulConstant(tanh_c) [-> deprocess] written as fp32 NCHW [3][outH][outW]
  int final_mode;  // 0 = raw, 1 = net space, 2 = fused vgg.deprocess
  float *out3;
  float tanh_c;
  // operand epilogue (batch-normalized nets; set_opnd_epilogue): instead of the raw output, acc * epi_scale + bias (+ReLU)
  // (+ the skip operand read at (y + epi_shave, x + epi_shave)) is split into fp16 hi / lo and stored at output (yo, xo),
  // channel epi_c0 + c of epi_dst, the next convolution's operand.  epi_c0: the N block's first channel.
  int opnd, epi_relu, epi_skip, epi_shave, epi_c0;
  const float *epi_scale;
  Operand epi_dst, epi_skip_op;  // per-image strides: Operand::img16
  // a batch of nimg images of one size (tile_at): image b of every tensor starts b * <stride> elements in -- the A operand
  // (16-byte units), raw (floats), out3 (floats), stats (doubles), nl_raw (float4 units), nl_sums (doubles)
  int nimg;
  int64_t a_img16, raw_img, out3_img, stats_img, nl_raw_img4, nl_sums_img;
  // the weights are packed multiplied by 2^w_exp (ConvDef::w_exp): every epilogue takes acc * w_unscale = acc * 2^-w_exp before
  // the bias.  The operand epilogue has it folded into epi_scale instead.
  float w_unscale;
};

// Tile T of a batched job, T = b * ntiles + t for image b and tile t of that image's output (0 <= T < nimg * ntiles): every role
// of conv_tc_kernel (consumers, patch / weight / norm-on-load producers) walks T = blockIdx.x, blockIdx.x + gridDim.x, ... and
// decodes it here, as does the CPU emulator (tests/emu/batch_emu.cu).  y / x0: the tile's output row and first output column;
// the rest: image b's base offsets into each tensor of the job.
struct TileAt {
  int b, y, x0;
  int64_t a16, raw, out3, stats, nl_raw4, nl_sums;  // the operand epilogue's: opnd_epi_addr
};
// batch == false: a single-image launch (nimg == 1, T = t), decoded without the division by ntiles
__host__ __device__ inline TileAt tile_at(const ConvJob &j, int T, bool batch = true) {
  TileAt a;
  a.b = batch ? T / j.ntiles : 0;
  const int t = T - a.b * j.ntiles;
  a.y = t / j.tiles_x;
  a.x0 = (t - a.y * j.tiles_x) * j.tile_dx;
  a.a16 = a.b * j.a_img16; a.raw = a.b * j.raw_img; a.out3 = a.b * j.out3_img; a.stats = a.b * j.stats_img;
  a.nl_raw4 = a.b * j.nl_raw_img4; a.nl_sums = a.b * j.nl_sums_img;
  return a;
}

// Operand epilogue addressing, shared by conv_tc_kernel and its CPU emulators (tests/emu/opnd_epi_emu.cu, batch_emu.cu).  tile:
// the batched tile index T of tile_at.  Consumer thread t (0..255) of a tile holds, for i < Npad / 8 and h < 2, the accumulator pair of channels c, c + 1 (c = 8i + 2 (t % 4)) of tile
// pixel r0 + 8h (r0 = 64 (t / 128) + 16 (t / 32 % 4) + t % 32 / 4).  Returns false when that pair lies outside the job's
// output (no store); else the 4-byte offsets of its fp16 pair in the hi / lo planes of epi_dst and, for a residual skip, of
// epi_skip_op.
__host__ __device__ inline bool opnd_epi_addr(const ConvJob &j, const TileAt &at, int t, int i, int h, int64_t &dst4, int64_t &skip4) {
  const int y = at.y, x = at.x0 + (t >> 7) * 64 + ((t >> 5) & 3) * 16 + ((t & 31) >> 2) + 8 * h;
  const int c = 8 * i + 2 * (t & 3);
  if (x >= j.Wo || y >= j.Ho || c >= j.Cout) return false;
  const int yo = y * j.oy_mul + j.oy_off, xo = x * j.ox_mul + j.ox_off;
  dst4 = at.b * j.epi_dst.img16 * 4 + j.epi_dst.pair_off4(yo, xo, j.epi_c0 + c);
  skip4 = j.epi_skip ? at.b * j.epi_skip_op.img16 * 4 + j.epi_skip_op.pair_off4(yo + j.epi_shave, xo + j.epi_shave, j.epi_c0 + c) : 0;
  return true;
}
__host__ __device__ inline bool opnd_epi_addr(const ConvJob &j, int tile, int t, int i, int h, int64_t &dst4, int64_t &skip4,
                                              bool batch = true) {
  return opnd_epi_addr(j, tile_at(j, tile, batch), t, i, h, dst4, skip4);
}

// Stacked-phase epilogue addressing (ConvJob::nstack > 0), shared by conv_tc_kernel and its CPU emulator
// (tests/emu/phase_stack_emu.cu).  Consumer thread t holds the accumulator pair of columns n, n + 1 (n = 8i + 2 (t % 4)) of tile
// pixel r0 + 8h, as in opnd_epi_addr.  They are channels c, c + 1 of phase s = n / Cout (Cout % 8 == 0, so s = 8i / Cout and
// both columns lie in one phase).  Returns false when the pixel lies outside the job's grid (no store); else the float offset
// of the pair in the image's raw output.
__host__ __device__ inline bool stack_epi_addr(const ConvJob &j, int y, int x0, int t, int i, int h, int64_t &raw_off) {
  const int s = 8 * i / j.Cout, c = 8 * i + 2 * (t & 3) - s * j.Cout;
  const int x = x0 + (t >> 7) * 64 + ((t >> 5) & 3) * 16 + ((t & 31) >> 2) + 8 * h;
  if (x >= j.Wo || y >= j.Ho || s >= j.nstack) return false;
  const int yo = y * j.oy_mul + j.st_oy[s], xo = x * j.ox_mul + j.st_ox[s];
  raw_off = (((int64_t)yo * j.raw_Cq + (c >> 2)) * j.raw_Wp + xo) * 4 + (c & 3);
  return true;
}
// Fused statistics: the per-warp partial sums are kept per accumulator column, and column n flushes into channel
// stats_channel(n) of the job's [sum][sum of squares] array (tc_flush_stats; columns >= stats_columns hold padding).  A stacked
// job thus sends each phase's partial sums out separately, the same float partials the one-job-per-phase plan sends, so the
// double totals -- and the normalised layer -- are the per-phase plan's.
__host__ __device__ inline int stats_columns(const ConvJob &j) { return j.nstack ? j.nstack * j.Cout : j.Cout; }
__host__ __device__ inline int stats_channel(const ConvJob &j, int n) { return j.nstack ? n % j.Cout : n; }

// Norm-on-load addressing, shared by the producer warps of conv_tc_kernel and their CPU emulator (tests/emu/nl_geom_emu.cu).
// The producer stages, for every patch pixel, the value the bulk copies would read from the operand that in_apply writes:
// patch row ri of group g is raw row nl_raw_row, pixel p of a (patch row, channel block) slab is raw column nl_raw_col, and
// a pixel outside [0, nl_H) x [0, nl_W) is zero (the operand's zero border).  One segment: storage column seg_src16[0] + x0 + p.
// Two segments (stride-2 consumers, parity-split operand [Cb][2][Ws2]): segment s is parity plane s, so its pixel
// p - seg_dst16[s] is storage column 2 (x0 + p - seg_dst16[s]) + s.
__host__ __device__ inline int nl_raw_row(const ConvJob &j, int y, int g, int ri) { return j.row_mul * y + j.grp_row[g][ri] - j.nl_padT; }
__host__ __device__ inline int nl_raw_col(const ConvJob &j, int x0, int p) {
  if (j.nseg == 1) return j.seg_src16[0] + x0 + p - j.nl_padL;
  const int s = p >= j.seg_dst16[1] ? 1 : 0;
  return 2 * (x0 + p - j.seg_dst16[s]) + s - j.nl_padL;
}
// the patch layouts the norm-on-load producer can fill (nl_raw_col): every pixel of a slab comes from one storage row, in one
// segment, or in the two parity segments of a stride-2 consumer
__host__ __device__ inline bool nl_geometry_ok(const ConvJob &j) {
  if (j.rf_R || j.pf || j.opnd || j.mt != 1) return false;
  if (j.nseg == 1) return j.seg_dst16[0] == 0 && j.seg_len16[0] == j.pslab16;
  return j.nseg == 2 && j.seg_src16[0] == 0 && j.seg_dst16[0] == 0 && j.seg_dst16[1] == j.seg_len16[0] &&
         j.seg_len16[0] + j.seg_len16[1] == j.pslab16 && j.seg_src16[1] == j.a_slab16 / 2;
}

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
// nimg > 1: a batch of images of one size -- in [nimg][Cin][H][W]; raw, operands and sums per image (RawTensor::img,
// Operand::img16, sums_img doubles apart)
int launch_pack_input(const float *in, int Cin, int H, int W, int reflect, const Operand &dst, cudaStream_t st, int nimg = 1);
int launch_in_stats(const RawTensor &raw, double *sums /*[2*C]*/, cudaStream_t st, int nimg = 1, int64_t sums_img = 0);
// sums == null: no normalisation (batch-normalized nets on the CUDA-core comparator: ReLU / skip / pack only)
int launch_in_apply(const RawTensor &raw, const double *sums, const float *gamma, const float *beta, float eps, int relu,
                    const Operand *skip, int shave, const Operand &dst, cudaStream_t st, int nimg = 1, int64_t sums_img = 0);
// tab_mean / tab_scale non-null: a fixed per-channel affine (inference-mode BatchNorm) instead of the statistics of src
int launch_up_in(const Operand &src, double *sums, const float *gamma, const float *beta, float eps, int relu, int scale,
                 const Operand &dst, cudaStream_t st, const float *tab_mean = nullptr, const float *tab_scale = nullptr,
                 int nimg = 1, int64_t sums_img = 0);
int launch_unpack_operand(const Operand &src, float *out_nchw, cudaStream_t st);

}  // namespace fav
