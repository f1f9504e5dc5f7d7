// conv_plan.hpp -- host-only planning of the wgmma implicit-GEMM convolution: filter-tap tables, K-step
// tables, weight packing and operand geometry.  Pure functions without CUDA runtime calls so that the same
// code is exercised on the CPU by tests/emu (an emulation of the kernel's addressing) and on the GPU by net.cu.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "conv.cuh"

namespace fav {

static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

struct Unit {  // one K8 unit of a K16 step: filter tap index (or -1 = zero weights) and input channel block
  int tap, cb;
};

struct ConvPhase {
  std::vector<ConvTap> taps;
  int oy_off = 0, ox_off = 0;
  // tcgen05 tables (size independent)
  int kind = 0;  // 0: stride-1 input, Cin_pad >= 16; 1: Cin_pad == 8 (tap pairing); 2: stride-2 parity-split input;
                 // 3: x-fold (filter columns folded into N; final wide conv with Cout <= 4)
  int Npad = 0;  // GEMM N of this phase
  int dxmin = 0, dxmax = 0;
  std::vector<int> rows;  // distinct dy, ascending
  int nrg = 1, nchg = 1, CbG = 1, rows_per_group = 1;
  int pslab16 = 0, nseg = 1, seg_len16[2] = {0, 0}, seg_dst16[2] = {0, 0};
  int nchunks = 1, spc = 1;
  int rf_R = 0, rf_rps = 0;                    // row-fold: output rows per unit, patch rows per stage (0 = off)
  int pf = 0;                                  // phase-fold (transposed conv): see conv.cuh
  // stacked job (plan_phase_stack): nstack sub-pixel phases along N, phase s at output offset (stack_oy[s], stack_ox[s]) in
  // columns [s Cout, (s + 1) Cout); its taps are the union of theirs (ky / kx unused).  0: an ordinary phase
  int nstack = 0, stack_oy[4] = {0, 0, 0, 0}, stack_ox[4] = {0, 0, 0, 0};
  std::vector<KStep> steps;                    // per group
  std::vector<std::vector<Unit>> units;        // [group][step*2 + u]
  float *d_w_simt = nullptr;
  uint4 *d_b_tc = nullptr;
};

struct ConvDef;
static inline int build_phase_fold(const ConvDef &c, struct ConvPhase &ph);

struct ConvDef {
  std::string name;
  int cin = 0, cout = 0, k = 0, stride = 1, pad = 0, adj = 0;
  bool transposed = false;
  int cin_pad = 0, Cb = 0, Npad = 0, cout_pad8 = 0;
  int in_stride = 1;  // stride of the input sampling grid (2 for 'd' layers)
  int tpad = 0;       // transposed: zero border the input operand needs (= -min tap offset over the sub-pixel phases)
  int out_mul = 1;    // 2 for transposed stride-2 (sub-pixel phases)
  // the output is read back as raw [Ho][Cq][Wp][4] by the next kernel: every conv of the loss network and every conv of the
  // stylization net but its last.  Such a conv never takes the x-fold plan, whose epilogue writes the net's final tanh image
  // through ConvJob::out3 instead of the raw output.
  bool raw_out = false;
  std::vector<ConvPhase> phases;
  ConvPhase fold;    // transposed conv: all 4 phases in one tcgen05 job (phase-fold); phases[] stay for the comparator
  bool has_fold = false;
  // Cout > kMaxNBlock (stylization net): the ConvDef of each N block (plan_conv_nblocks); the tensor-core jobs come from
  // these, the CUDA-core comparator keeps the whole convolution's phases.  Empty: one job per phase of this ConvDef.
  std::vector<ConvDef> nblock;
  // stride-2 transposed conv with 2 Cout <= 128 (plan_phase_stack): the tensor-core jobs with the sub-pixel phases stacked
  // along N, and their bias (the layer's, once per stacked phase).  Empty: one job per phase.
  std::vector<ConvPhase> stack;
  float *d_stack_bias = nullptr;
  float *d_bias = nullptr;
  float *d_scale = nullptr;  // batch-normalized nets: the per-channel BN scale the operand epilogue applies (Npad floats)
  int pw = -1, pb = -1;  // param indices
};

// ---- tcgen05 tables for one phase -------------------------------------------------------------------------
static constexpr int kStageCapBytes = 56 * 1024;  // one A stage (hi + lo)
static constexpr int kChunkCapBytes = 24 * 1024;
// conv_tc.cu (wgmma) keeps one register accumulator of Npad columns per 64-pixel half-tile.  The row-fold and phase-fold
// plans write per-row / per-phase column ranges of one wide accumulator, two-row units and the K-split need a second
// accumulator: none of them is planned.
static constexpr bool kPlanRowFold = false, kPlanPhaseFold = false;

static inline int build_phase_tables(const ConvDef &c, ConvPhase &ph) {
  // a transposed conv whose stride exceeds its kernel (f1s2) leaves sub-pixel phases that only receive the bias: no K steps to
  // plan, and no released model has one
  if (ph.taps.empty()) {
    set_error("conv %s: sub-pixel phase (%d,%d) without filter taps (kernel %d smaller than stride %d)", c.name.c_str(),
              ph.oy_off, ph.ox_off, c.k, c.stride);
    return FAV_ERR_UNSUPPORTED;
  }
  ph.rows.clear();
  ph.dxmin = 1 << 30; ph.dxmax = -(1 << 30);
  for (auto &t : ph.taps) {
    if (std::find(ph.rows.begin(), ph.rows.end(), t.dy) == ph.rows.end()) ph.rows.push_back(t.dy);
    ph.dxmin = std::min(ph.dxmin, t.dx); ph.dxmax = std::max(ph.dxmax, t.dx);
  }
  std::sort(ph.rows.begin(), ph.rows.end());
  std::vector<int> dxs;
  for (int dx = ph.dxmin; dx <= ph.dxmax; ++dx) dxs.push_back(dx);
  auto tap_index = [&](int dy, int dx) {
    for (size_t i = 0; i < ph.taps.size(); ++i)
      if (ph.taps[i].dy == dy && ph.taps[i].dx == dx) return (int)i;
    return -1;
  };
  const int nrows = (int)ph.rows.size();
  ph.Npad = ph.nstack ? round_up(ph.nstack * c.cout, 16) : c.Npad;
  const bool xfold = !c.raw_out && !c.transposed && c.in_stride == 1 && c.k >= 5 && c.cout <= 4 && c.Cb % 2 == 0 && c.pad == (c.k - 1) / 2;
  if (xfold) {
    ph.kind = 3; ph.Npad = round_up(c.k * c.cout, 16);
    ph.CbG = (c.Cb % 4 == 0) ? 4 : 2; ph.nchg = c.Cb / ph.CbG;
    ph.nseg = 1; ph.pslab16 = kTileM; ph.seg_len16[0] = kTileM; ph.seg_dst16[0] = 0;
    ph.nrg = 0;
    for (int rg = 1; rg <= nrows; ++rg) {
      if (nrows % rg) continue;
      if ((nrows / rg) * ph.CbG * ph.pslab16 * 32 <= kStageCapBytes) { ph.nrg = rg; break; }
    }
    if (!ph.nrg) { set_error("conv %s: patch stage too large", c.name.c_str()); return FAV_ERR_UNSUPPORTED; }
    ph.rows_per_group = nrows / ph.nrg;
  } else if (c.in_stride == 2) {
    if (!(c.k == 3 && c.pad == 1 && c.Cb >= 2 && c.Cb % 2 == 0)) {
      set_error("conv %s: stride-2 tcgen05 path needs k=3, pad=1, Cin%%16==0", c.name.c_str());
      return FAV_ERR_UNSUPPORTED;
    }
    ph.kind = 2; ph.CbG = 2; ph.nchg = c.Cb / 2; ph.nrg = 1; ph.rows_per_group = nrows;
    ph.nseg = 2; ph.seg_len16[0] = kTileM + 1; ph.seg_dst16[0] = 0; ph.seg_len16[1] = kTileM; ph.seg_dst16[1] = kTileM + 1;
    ph.pslab16 = 2 * kTileM + 1;
  } else if (c.cin_pad == 8) {
    ph.kind = 1; ph.CbG = 1; ph.nchg = 1; ph.nrg = 1; ph.rows_per_group = nrows;
    int ntx = (int)dxs.size(), ntx_pad = round_up(ntx, 2);
    ph.nseg = 1; ph.pslab16 = kTileM + ntx_pad; ph.seg_len16[0] = ph.pslab16; ph.seg_dst16[0] = 0;
  } else {
    if (c.Cb % 2) {
      set_error("conv %s: Cin must be 8 or a multiple of 16 for the tcgen05 path", c.name.c_str());
      return FAV_ERR_UNSUPPORTED;
    }
    ph.kind = 0; ph.CbG = (c.Cb % 4 == 0) ? 4 : 2;
    if (const char *e = getenv("FAV_CBG")) { int v = atoi(e); if (v == 2 || v == 4) ph.CbG = v; }  // tuning knob
    ph.nchg = c.Cb / ph.CbG;
    ph.nseg = 1; ph.pslab16 = kTileM + (ph.dxmax - ph.dxmin); ph.seg_len16[0] = ph.pslab16; ph.seg_dst16[0] = 0;
    ph.nrg = 0;
    for (int rg = 1; rg <= nrows; ++rg) {
      if (nrows % rg) continue;
      if ((nrows / rg) * ph.CbG * ph.pslab16 * 32 <= kStageCapBytes) { ph.nrg = rg; break; }
    }
    if (!ph.nrg) { set_error("conv %s: patch stage too large", c.name.c_str()); return FAV_ERR_UNSUPPORTED; }
    ph.rows_per_group = nrows / ph.nrg;
  }
  if (ph.rows_per_group * ph.CbG * ph.pslab16 * 32 > kStageCapBytes || ph.rows_per_group > kMaxRows ||
      ph.nrg * ph.nchg > kMaxGroups) {
    set_error("conv %s: tcgen05 tiling limits exceeded", c.name.c_str());
    return FAV_ERR_UNSUPPORTED;
  }
  // steps of one group (identical for every group) + per-group unit lists
  ph.steps.clear();
  const int ngroups = ph.nrg * ph.nchg;
  ph.units.assign(ngroups, {});
  for (int ri = 0; ri < ph.rows_per_group; ++ri) {
    if (ph.kind == 1) {
      for (int p = 0; p * 2 < (int)dxs.size(); ++p) {
        ph.steps.push_back(KStep{(uint16_t)(ri * ph.pslab16 + 2 * p), 1});
        for (int g = 0; g < ngroups; ++g)
          for (int u = 0; u < 2; ++u) {
            int di = 2 * p + u;
            int tap = di < (int)dxs.size() ? tap_index(ph.rows[ri], dxs[di]) : -1;
            ph.units[g].push_back(Unit{tap, 0});
          }
      }
    } else if (ph.kind == 3) {
      for (int j = 0; j < ph.CbG / 2; ++j) {
        ph.steps.push_back(KStep{(uint16_t)((ri * ph.CbG + 2 * j) * ph.pslab16), (uint16_t)ph.pslab16});
        for (int chg = 0; chg < ph.nchg; ++chg)
          for (int rg = 0; rg < ph.nrg; ++rg) {
            int g = chg * ph.nrg + rg;
            int ky = ph.rows[rg * ph.rows_per_group + ri] + c.pad;  // unit.tap holds the filter ROW in x-fold mode
            for (int u = 0; u < 2; ++u) ph.units[g].push_back(Unit{ky, chg * ph.CbG + 2 * j + u});
          }
      }
    } else {
      for (int dx : dxs) {
        int xoff = ph.kind == 2 ? (dx == -1 ? 0 : (dx == 0 ? kTileM + 1 : 1)) : dx - ph.dxmin;
        for (int j = 0; j < ph.CbG / 2; ++j) {
          ph.steps.push_back(KStep{(uint16_t)((ri * ph.CbG + 2 * j) * ph.pslab16 + xoff), (uint16_t)ph.pslab16});
          for (int chg = 0; chg < ph.nchg; ++chg)
            for (int rg = 0; rg < ph.nrg; ++rg) {
              int g = chg * ph.nrg + rg;
              int tap = tap_index(ph.rows[rg * ph.rows_per_group + ri], dx);
              for (int u = 0; u < 2; ++u) ph.units[g].push_back(Unit{tap, chg * ph.CbG + 2 * j + u});
            }
        }
      }
    }
  }
  // ---- row-fold for tall filters with a narrow N block (see conv.cuh) -------------------------------------------
  ph.rf_R = 0;
  if (kPlanRowFold && (ph.kind == 1 || ph.kind == 3) && !c.transposed && c.in_stride == 1 && nrows >= 5 && ph.Npad <= 32 &&
      nrows * ph.Npad <= 512 && c.Cb <= 4) {  // Cb = 8 (64-channel final conv of the paper arch): a 35 KB patch row per
                                              // stage leaves 12 MMAs per stage -- latency bound, 359 us vs 156 us unfolded (measured)
    const int saveCbG = ph.CbG, saveNchg = ph.nchg;
    ph.CbG = c.Cb; ph.nchg = 1;  // a row stage holds every channel block of the patch row
    bool consecutive = true;
    for (size_t i = 1; i < ph.rows.size(); ++i) consecutive = consecutive && ph.rows[i] == ph.rows[i - 1] + 1;
    // R output rows per unit: the patch-row re-read factor is (R + KH - 1) / R.  The wide-input x-fold layer (final conv)
    // is bound by that L2 -> SM traffic, so it takes R = 8 (8 x 32 = 256 accumulator columns, still double buffered);
    // conv1 (one channel block) is issue bound and keeps R = 4 so that the unit can be K-split between two warps.
    int cand[2] = {(ph.kind == 3 && 8 * ph.Npad <= 256) ? 8 : 4, 4};
    if (const char *e = getenv(ph.kind == 3 ? "FAV_RF_R3" : "FAV_RF_R1")) cand[0] = cand[1] = atoi(e);
    const int row_bytes = ph.CbG * ph.pslab16 * 32;  // hi + lo of one patch row
    int R = 0, rps = 0, total_rows = 0;
    for (int ci = 0; ci < 2 && rps == 0; ++ci) {
      R = cand[ci]; total_rows = R + nrows - 1;
      for (int d = total_rows; d >= 1; --d)
        if (total_rows % d == 0 && total_rows / d <= kMaxGroups && d <= kMaxRows && d * row_bytes <= 36 * 1024) { rps = d; break; }
    }
    if (consecutive && rps > 0) {
      ph.rf_R = R; ph.rf_rps = rps;
      // K steps of ONE patch row; units hold (tap column or channel block) only -- the filter row comes from iy - r
      ph.steps.clear();
      ph.units.assign(1, {});
      if (ph.kind == 1) {
        for (int p = 0; p * 2 < (int)dxs.size(); ++p) {
          ph.steps.push_back(KStep{(uint16_t)(2 * p), 1});
          for (int u = 0; u < 2; ++u) ph.units[0].push_back(Unit{2 * p + u < (int)dxs.size() ? 2 * p + u : -1, 0});  // tap = kx
        }
      } else {
        for (int j = 0; j < ph.CbG / 2; ++j) {
          ph.steps.push_back(KStep{(uint16_t)(2 * j * ph.pslab16), (uint16_t)ph.pslab16});
          for (int u = 0; u < 2; ++u) ph.units[0].push_back(Unit{0, 2 * j + u});
        }
      }
      ph.nrg = 1; ph.rows_per_group = rps;
      ph.spc = (int)ph.steps.size(); ph.nchunks = 1;  // weights: one resident image (see pack_phase_weights)
      return FAV_OK;
    }
    ph.CbG = saveCbG; ph.nchg = saveNchg;
  }
  const int spg = (int)ph.steps.size();
  if (spg > kMaxSteps) { set_error("conv %s: too many K steps", c.name.c_str()); return FAV_ERR_UNSUPPORTED; }
  const int step_bytes = 2 * 2 * ph.Npad * 16;
  ph.spc = 1;
  for (int d = 1; d <= spg; ++d)
    if (spg % d == 0 && d * step_bytes <= kChunkCapBytes && d <= 8) ph.spc = d;  // 8 = kMaxSpc of conv_tc.cu
  ph.nchunks = spg / ph.spc;
  return FAV_OK;
}

static inline uint16_t f2h_bits(float f) {
  __half h = __float2half_rn(f);
  uint16_t b;
  memcpy(&b, &h, 2);
  return b;
}
static inline float h2f_bits(uint16_t b) {
  __half h;
  memcpy(&h, &b, 2);
  return __half2float(h);
}

static inline float weight_at(const ConvDef &c, const std::vector<float> &w, int co, int ci, int ky, int kx) {
  if (co >= c.cout || ci >= c.cin) return 0.f;
  if (c.transposed) return w[(((int64_t)ci * c.cout + co) * c.k + ky) * c.k + kx];
  return w[(((int64_t)co * c.cin + ci) * c.k + ky) * c.k + kx];
}


// ---- phase-fold ---------------------------------------------------------------------------------------------------
static const int kPfA[4] = {0, 0, 1, 1}, kPfB[4] = {0, 1, 1, 0};               // block -> phase (a,b)
static const int kPfTapDy[4] = {0, 0, 1, 1}, kPfTapDx[4] = {0, 1, 0, 1};       // chunk -> tap (dy,dx)
static const int kPfBlk0[4] = {0, 1, 2, 2}, kPfNblk[4] = {4, 2, 2, 1};         // chunk -> first block, #blocks

static inline int build_phase_fold(const ConvDef &c, ConvPhase &ph) {
  if (!(c.transposed && c.k == 3 && c.stride == 2 && c.pad == 1 && c.adj == 1 && c.Cb % 2 == 0 && c.cout % 16 == 0 &&
        4 * c.cout <= 256))
    return FAV_ERR_UNSUPPORTED;
  ph.pf = 1; ph.kind = 0; ph.Npad = 4 * c.cout;
  ph.taps.clear();
  for (int t = 0; t < 4; ++t) ph.taps.push_back(ConvTap{kPfTapDy[t], kPfTapDx[t], 0, 0});
  ph.rows = {0, 1}; ph.dxmin = 0; ph.dxmax = 1;
  ph.CbG = (c.Cb % 4 == 0) ? 4 : 2; ph.nchg = c.Cb / ph.CbG; ph.nrg = 1; ph.rows_per_group = 2;
  ph.nseg = 1; ph.pslab16 = kTileM + 1; ph.seg_len16[0] = ph.pslab16; ph.seg_dst16[0] = 0;
  ph.steps.clear();
  for (int t = 0; t < 4; ++t)
    for (int j = 0; j < ph.CbG / 2; ++j)
      ph.steps.push_back(KStep{(uint16_t)((kPfTapDy[t] * ph.CbG + 2 * j) * ph.pslab16 + kPfTapDx[t]), (uint16_t)ph.pslab16});
  ph.spc = ph.CbG / 2; ph.nchunks = 4;
  return FAV_OK;
}

// weights of the folded job: [group][tap chunk][hi|lo][pair][k-half][n = blk*Cout + co][8]
static inline std::vector<uint16_t> pack_phase_fold(const ConvDef &c, const ConvPhase &ph, const std::vector<float> &w) {
  const int spc = ph.CbG / 2;
  size_t grp = 0;
  for (int t = 0; t < 4; ++t) grp += (size_t)2 * spc * 2 * kPfNblk[t] * c.cout * 8;
  std::vector<uint16_t> pk((size_t)ph.nchg * grp, 0);
  for (int g = 0; g < ph.nchg; ++g) {
    size_t base = (size_t)g * grp;
    for (int t = 0; t < 4; ++t) {
      const int n = kPfNblk[t] * c.cout;
      for (int part = 0; part < 2; ++part)
        for (int j = 0; j < spc; ++j)
          for (int u = 0; u < 2; ++u) {
            const int cb = g * ph.CbG + 2 * j + u;
            for (int bi = 0; bi < kPfNblk[t]; ++bi) {
              const int blk = kPfBlk0[t] + bi, a = kPfA[blk], b = kPfB[blk];
              const int ky = a + c.pad - 2 * kPfTapDy[t], kx = b + c.pad - 2 * kPfTapDx[t];  // oy = 2*iy - pad + ky
              for (int co = 0; co < c.cout; ++co)
                for (int i = 0; i < 8; ++i) {
                  float v = (ky >= 0 && ky < c.k && kx >= 0 && kx < c.k) ? weight_at(c, w, co, cb * 8 + i, ky, kx) : 0.f;
                  uint16_t hb = f2h_bits(v);
                  size_t o = base + ((((size_t)part * spc + j) * 2 + u) * n + (size_t)bi * c.cout + co) * 8 + i;
                  pk[o] = part == 0 ? hb : f2h_bits(v - h2f_bits(hb));
                }
            }
          }
      base += (size_t)2 * spc * 2 * n * 8;
    }
  }
  return pk;
}

// taps of a plain convolution / the 4 sub-pixel phases of a stride-2 transposed convolution
static inline void build_phases(ConvDef &c) {
  c.phases.clear();
  if (!c.transposed) {
    ConvPhase ph;
    for (int ky = 0; ky < c.k; ++ky)
      for (int kx = 0; kx < c.k; ++kx) ph.taps.push_back(ConvTap{ky - c.pad, kx - c.pad, ky, kx});
    c.phases.push_back(std::move(ph));
  } else {
    // out[s*y+a, s*x+b]:  oy = s*iy - pad + ky  =>  s*iy = s*y + (a + pad - ky): one sub-pixel phase per (a, b), its taps are
    // the filter taps with (a + pad - ky) divisible by the stride (stride 1, the fXs1 token: a plain convolution with the
    // flipped filter)
    const int sdiv = c.stride;
    auto fdiv = [](int n, int d) { return n >= 0 ? n / d : -((-n + d - 1) / d); };
    c.tpad = 0;
    for (int a = 0; a < sdiv; ++a)
      for (int b = 0; b < sdiv; ++b) {
        ConvPhase ph;
        ph.oy_off = a; ph.ox_off = b;
        for (int ky = 0; ky < c.k; ++ky) {
          int ny = a + c.pad - ky;
          if (((ny % sdiv) + sdiv) % sdiv) continue;
          for (int kx = 0; kx < c.k; ++kx) {
            int nx = b + c.pad - kx;
            if (((nx % sdiv) + sdiv) % sdiv) continue;
            ph.taps.push_back(ConvTap{fdiv(ny, sdiv), fdiv(nx, sdiv), ky, kx});
            c.tpad = std::max(c.tpad, std::max(-fdiv(ny, sdiv), -fdiv(nx, sdiv)));
          }
        }
        c.phases.push_back(std::move(ph));
      }
    c.has_fold = kPlanPhaseFold && build_phase_fold(c, c.fold) == FAV_OK;
  }
}

static inline void init_conv_def(ConvDef &c, const std::string &name, int cin, int cout, int k, int stride, int pad,
                                 bool tr, int adj) {
  c.name = name; c.cin = cin; c.cout = cout; c.k = k; c.stride = stride; c.pad = pad; c.transposed = tr; c.adj = adj;
  c.cin_pad = round_up(cin, 8);
  c.Cb = c.cin_pad / 8;
  c.Npad = std::max(16, round_up(cout, 16));
  c.cout_pad8 = round_up(cout, 8);
  c.in_stride = (!tr && stride == 2) ? 2 : 1;
  c.out_mul = tr ? stride : 1;
}

// ---- N blocks: a convolution with Cout > kMaxNBlock runs as ceil(Cout / 128) jobs of <= 128 output channels each (per
// sub-pixel phase, for a transposed convolution).  Block b is an ordinary convolution over every input channel with output
// channels [128 b, 128 b + cout_b): its own ConvDef (so its own tables and packed weights), a bias slice, a raw output
// pointer advanced by 128 b channels (32 b channel quads of the [Ho][Cq][Wp][4] layout; the row pitch Cq stays the full
// tensor's) and, in the stylization net, the fused InstanceNorm statistics of those channels (conv_nblock_stats).
static inline int conv_nblocks(int cout) { return (cout + kMaxNBlock - 1) / kMaxNBlock; }
static inline int conv_nblock_cout(int cout, int b) { return std::min(kMaxNBlock, cout - b * kMaxNBlock); }
// weights [Cout][Cin][k][k] -> the [cout_b][Cin][k][k] slice of block b; transposed weights [Cin][Cout][k][k] (Torch's
// SpatialFullConvolution layout) -> the [Cin][cout_b][k][k] slice
static inline std::vector<float> conv_nblock_weights(const std::vector<float> &w, int cin, int cout, int k, int b,
                                                     bool transposed = false) {
  const size_t kk = (size_t)k * k, c0 = (size_t)b * kMaxNBlock, n = (size_t)conv_nblock_cout(cout, b);
  if (!transposed) return std::vector<float>(w.begin() + c0 * cin * kk, w.begin() + (c0 + n) * cin * kk);
  std::vector<float> s;
  s.reserve((size_t)cin * n * kk);
  for (int ci = 0; ci < cin; ++ci) {
    const auto first = w.begin() + ((size_t)ci * cout + c0) * kk;
    s.insert(s.end(), first, first + n * kk);
  }
  return s;
}
// the ConvDef of N block b (raw output, so never the x-fold plan)
static inline void init_nblock_conv_def(ConvDef &c, const std::string &name, int cin, int cout, int k, int stride, int pad, int b,
                                        bool transposed = false, int adj = 0) {
  init_conv_def(c, name, cin, conv_nblock_cout(cout, b), k, stride, pad, transposed, adj);
  c.raw_out = true;
  build_phases(c);
}
static inline int64_t conv_nblock_raw_offset(int b, int raw_Wp) { return (int64_t)b * (kMaxNBlock / 4) * raw_Wp * 4; }
// fused InstanceNorm statistics of block b: sums = the whole tensor's [sum][sum of squares] array of cout channels each; the
// epilogue adds channel c of the block into job.stats[c] and job.stats[job.stats_pitch + c]
static inline void conv_nblock_stats(ConvJob &j, double *sums, int cout, int b) {
  j.stats = sums ? sums + (int64_t)b * kMaxNBlock : nullptr;
  j.stats_pitch = cout;
}
// operand epilogue of a batch-normalized net's non-final convolution: job j of N block b writes acc * scale + bias (+ReLU)
// (+skip: the block input `skip` shifted by `shave`) straight into `dst`, the next convolution's operand (opnd_epi_addr,
// conv.cuh).  scale: the block's per-channel BN scale, bias the folded bias.  No raw output, no statistics.
static inline void set_opnd_epilogue(ConvJob &j, int b, const float *scale, const Operand &dst, int relu, const Operand *skip,
                                     int shave) {
  j.opnd = 1; j.epi_scale = scale; j.epi_c0 = b * kMaxNBlock; j.epi_dst = dst; j.epi_relu = relu;
  j.epi_skip = skip ? 1 : 0; j.epi_skip_op = skip ? *skip : Operand(); j.epi_shave = skip ? shave : 0;
  j.raw = nullptr; j.stats = nullptr;
}
// norm-on-load (conv_tc.cu): job j reads `raw`, the raw output of the previous convolution, and applies its InstanceNorm
// (+ReLU) and the fp16 hi / lo split while it stages the patch, instead of reading `in`, the operand in_apply would write from
// it (nl_raw_row / nl_raw_col, conv.cuh).  sums: raw's fused statistics, sums_img doubles apart per image.
static inline void set_norm_on_load(ConvJob &j, const RawTensor &raw, const Operand &in, int relu, const double *sums,
                                    int64_t sums_img, const float *gamma, const float *beta) {
  j.nl = 1;
  j.nl_raw = reinterpret_cast<const float4 *>(raw.p); j.nl_Cq = raw.Cq; j.nl_Wp = raw.Wp; j.nl_H = raw.H; j.nl_W = raw.W;
  j.nl_padT = in.padT; j.nl_padL = in.padL; j.nl_relu = relu; j.nl_C = raw.C;
  j.nl_sums = sums; j.nl_gamma = gamma; j.nl_beta = beta;
  j.nl_raw_img4 = raw.img / 4; j.nl_sums_img = sums_img;
  j.nl_inv_count = 1.0 / ((double)raw.H * raw.W); j.nl_eps = 1e-5;  // InstanceNormalization.lua:21
}
// a batch of nimg images of one size (conv.cuh tile_at): per-image strides of the job's raw output (floats), final frame (floats)
// and fused statistics (doubles); the A operand's and the operand epilogue's come with their Operands (Operand::img16)
static inline void set_conv_batch(ConvJob &j, int nimg, int64_t raw_img, int64_t out3_img, int64_t stats_img) {
  j.nimg = nimg; j.raw_img = raw_img; j.out3_img = out3_img; j.stats_img = stats_img;
}
// K-step tables of every phase of a stylization-net convolution, or of every N block's phases when Cout > kMaxNBlock.  A
// geometry the tensor-core planner cannot run fails here with FAV_ERR_UNSUPPORTED and the layer's name.
static inline int plan_conv_nblocks(ConvDef &c) {
  c.nblock.clear();
  if (conv_nblocks(c.cout) == 1) {
    for (ConvPhase &ph : c.phases) FAV_TRY(build_phase_tables(c, ph));
    return FAV_OK;
  }
  for (int b = 0; b < conv_nblocks(c.cout); ++b) {
    ConvDef cb;
    init_nblock_conv_def(cb, c.name, c.cin, c.cout, c.k, c.stride, c.pad, b, c.transposed, c.adj);
    for (ConvPhase &ph : cb.phases) FAV_TRY(build_phase_tables(cb, ph));
    c.nblock.push_back(std::move(cb));
  }
  return FAV_OK;
}

// ---- stacked sub-pixel phases: the phases of a stride-2 transposed conv share their input pixels, only the weights and the
// output placement differ.  So as many phases as fit N <= 128 run as one stride-1 conv over the input grid, phase s in columns
// [s Cout, (s + 1) Cout): all four when 4 Cout <= 128, else the two column phases b = 0, 1 of each row phase a.  The job's taps
// are the union of its phases' taps; where a tap does not feed phase s its weights are zero (extra MMA work, the useful FLOPs
// are unchanged).  Cout % 8 == 0 keeps each epilogue column pair inside one phase (stack_epi_addr).  c.phases stay as they
// are for the CUDA-core comparator and for batch-normalized nets, whose operand epilogue runs one phase per job.
static inline int plan_phase_stack(ConvDef &c) {
  c.stack.clear();
  if (!c.transposed || c.stride != 2 || c.cout % 8 || 2 * c.cout > kMaxNBlock) return FAV_OK;
  const int per_job = 4 * c.cout <= kMaxNBlock ? 4 : 2;  // c.phases: (a, b) = (0,0), (0,1), (1,0), (1,1)
  for (int p0 = 0; p0 < 4; p0 += per_job) {
    ConvPhase ph;
    ph.nstack = per_job;
    for (int s = 0; s < per_job; ++s) {
      const ConvPhase &p = c.phases[p0 + s];
      ph.stack_oy[s] = p.oy_off; ph.stack_ox[s] = p.ox_off;
      for (const ConvTap &t : p.taps) {
        bool have = false;
        for (const ConvTap &u : ph.taps) have = have || (u.dy == t.dy && u.dx == t.dx);
        if (!have) ph.taps.push_back(ConvTap{t.dy, t.dx, -1, -1});
      }
    }
    FAV_TRY(build_phase_tables(c, ph));
    c.stack.push_back(std::move(ph));
  }
  return FAV_OK;
}
// the bias of a stacked job (Npad floats): column s * Cout + co holds the layer's bias of channel co
static inline std::vector<float> stack_bias(const ConvDef &c, const std::vector<float> &b) {
  const ConvPhase &ph = c.stack[0];
  std::vector<float> sb(ph.Npad, 0.f);
  for (int n = 0; n < ph.nstack * c.cout; ++n) sb[n] = b[n % c.cout];
  return sb;
}

// packed tcgen05 weights of one phase: [group][chunk][hi|lo][step][k8 half][Npad][8] fp16 (as uint16 bit patterns)
static inline std::vector<uint16_t> pack_phase_weights(const ConvDef &c, const ConvPhase &ph, const std::vector<float> &w) {
  if (ph.rf_R) {
    // row-fold image: [step][hi|lo][k-half][n = (KH-1-ky)*Nblk + cblk][8], loaded once per CTA (one chunk per step)
    const int KH = (int)ph.rows.size(), Nblk = ph.Npad, NR = KH * Nblk, nst = (int)ph.steps.size();
    std::vector<uint16_t> pk((size_t)nst * 2 * 2 * NR * 8, 0);
    for (int st = 0; st < nst; ++st)
      for (int part = 0; part < 2; ++part)
        for (int u = 0; u < 2; ++u) {
          const Unit un = ph.units[0][st * 2 + u];
          if (un.tap < 0) continue;
          for (int ky = 0; ky < KH; ++ky)
            for (int cblk = 0; cblk < Nblk; ++cblk)
              for (int i = 0; i < 8; ++i) {
                float v;
                if (ph.kind == 3) {  // x-fold: cblk = kx * Cout + co
                  int kx = cblk / c.cout, co = cblk % c.cout;
                  v = kx < c.k ? weight_at(c, w, co, un.cb * 8 + i, ky, kx) : 0.f;
                } else {              // kind 1: unit.tap = kx, cblk = co
                  v = weight_at(c, w, cblk, i, ky, un.tap);
                }
                uint16_t hb = f2h_bits(v);
                size_t o = ((((size_t)st * 2 + part) * 2 + u) * NR + (size_t)(KH - 1 - ky) * Nblk + cblk) * 8 + i;
                pk[o] = part == 0 ? hb : f2h_bits(v - h2f_bits(hb));
              }
        }
    return pk;
  }
  const int ngroups = ph.nrg * ph.nchg, spg = (int)ph.steps.size();
  const int Npad = ph.Npad;
  std::vector<uint16_t> pk((size_t)ngroups * spg * 2 * 2 * Npad * 8, 0);
  for (int g = 0; g < ngroups; ++g)
    for (int ch = 0; ch < ph.nchunks; ++ch)
      for (int part = 0; part < 2; ++part)
        for (int st = 0; st < ph.spc; ++st)
          for (int u = 0; u < 2; ++u) {
            const Unit un = ph.units[g][(ch * ph.spc + st) * 2 + u];
            size_t base = (((((size_t)g * ph.nchunks + ch) * 2 + part) * ph.spc + st) * 2 + u) * Npad * 8;
            if (un.tap < 0) continue;
            for (int n = 0; n < Npad; ++n)
              for (int i = 0; i < 8; ++i) {
                float v;
                if (ph.kind == 3) {  // n = kx * Cout + co, unit.tap = ky
                  int kx = n / c.cout, co = n % c.cout;
                  v = kx < c.k ? weight_at(c, w, co, un.cb * 8 + i, un.tap, kx) : 0.f;
                } else if (ph.nstack) {  // n = s * Cout + co; tap (dy, dx) of phase (a, b) is filter tap (a + pad - 2 dy, b + pad - 2 dx)
                  const int s = n / c.cout, co = n % c.cout;
                  const int ky = s < ph.nstack ? ph.stack_oy[s] + c.pad - c.stride * ph.taps[un.tap].dy : -1;
                  const int kx = s < ph.nstack ? ph.stack_ox[s] + c.pad - c.stride * ph.taps[un.tap].dx : -1;
                  v = ky >= 0 && ky < c.k && kx >= 0 && kx < c.k ? weight_at(c, w, co, un.cb * 8 + i, ky, kx) : 0.f;
                } else {
                  v = weight_at(c, w, n, un.cb * 8 + i, ph.taps[un.tap].ky, ph.taps[un.tap].kx);
                }
                uint16_t hb = f2h_bits(v);
                pk[base + (size_t)n * 8 + i] = part == 0 ? hb : f2h_bits(v - h2f_bits(hb));
              }
          }
  return pk;
}

// geometry of the operand feeding convolution `consumer` (pointers left null)
static inline Operand operand_geometry(int C, int H, int W, const ConvDef *consumer) {
  Operand o;
  o.C = C; o.Cb = round_up(C, 8) / 8; o.H = H; o.W = W;
  int pad = consumer ? consumer->pad : 0;
  if (consumer && consumer->transposed) pad = consumer->tpad;
  o.padT = o.padL = pad;
  o.Hs = H + 2 * pad + 2 + 4;  // +2: transposed-conv / mt=2 overrun, +4: row-fold units of 4 output rows
  o.parity = (consumer && consumer->in_stride == 2) ? 1 : 0;
  o.Ws = pad + round_up(W, kTileM) + pad + 16;
  if (o.parity) o.Ws2 = round_up((W + 2 * pad + 1) / 2, kTileM) + 8;
  o.elems16 = (size_t)o.Hs * o.Cb * o.slab16() + 512;
  return o;
}

static inline void conv_out_size(const ConvDef &c, int H, int W, int *Ho, int *Wo) {
  if (c.transposed) {
    *Ho = (H - 1) * c.stride - 2 * c.pad + c.k + c.adj;
    *Wo = (W - 1) * c.stride - 2 * c.pad + c.k + c.adj;
  } else {
    *Ho = (H + 2 * c.pad - c.k) / c.stride + 1;
    *Wo = (W + 2 * c.pad - c.k) / c.stride + 1;
  }
}

// the device job of one phase (weights / bias / raw pointers filled by the caller)
static inline int fill_conv_job(const ConvDef &c, const ConvPhase &ph, const Operand &in, ConvJob &j) {
  int Ho, Wo;
  conv_out_size(c, in.H, in.W, &Ho, &Wo);
  const int pHo = c.transposed ? in.H : Ho, pWo = c.transposed ? in.W : Wo;  // phase grid
  memset(&j, 0, sizeof(j));
  j.nimg = 1; j.a_img16 = in.img16;
  j.a_hi = reinterpret_cast<const uint4 *>(in.hi); j.a_lo = reinterpret_cast<const uint4 *>(in.lo);
  j.a_Cb = in.Cb; j.a_slab16 = in.slab16();
  j.tile_dx = ph.kind == 3 ? kTileM - (c.k - 1) : kTileM;
  j.xfold_kw = ph.kind == 3 ? c.k : 0;
  j.mt = 1;  // one output row per unit (see kPlanRowFold)
  if (ph.rf_R) j.mt = ph.rf_R;
  if (ph.pf) j.mt = 1;
  j.Ho = pHo; j.Wo = pWo; j.tiles_x = ceil_div(pWo, j.tile_dx); j.ntiles = j.tiles_x * ceil_div(pHo, j.mt);
  j.row_mul = c.in_stride;
  j.nseg = ph.nseg;
  for (int s = 0; s < ph.nseg; ++s) { j.seg_len16[s] = ph.seg_len16[s]; j.seg_dst16[s] = ph.seg_dst16[s]; }
  if (ph.kind == 2) { j.seg_src16[0] = 0; j.seg_src16[1] = in.Ws2; }
  else j.seg_src16[0] = in.padL + ph.dxmin;
  j.ngroups = ph.nrg * ph.nchg; j.nrows = ph.rows_per_group; j.CbG = ph.CbG;
  for (int chg = 0; chg < ph.nchg; ++chg)
    for (int rg = 0; rg < ph.nrg; ++rg) {
      int g = chg * ph.nrg + rg;
      j.grp_cb0[g] = chg * ph.CbG;
      for (int ri = 0; ri < ph.rows_per_group; ++ri) j.grp_row[g][ri] = in.padT + ph.rows[rg * ph.rows_per_group + ri];
      if (j.mt == 2) j.grp_row[g][ph.rows_per_group] = j.grp_row[g][ph.rows_per_group - 1] + 1;
    }
  j.nrows = ph.rows_per_group + (j.mt - 1);  // patch rows per stage
  if (ph.rf_R) {  // stages = groups of rf_rps consecutive patch rows
    const int KH = (int)ph.rows.size();
    j.rf_R = ph.rf_R; j.rf_kh = KH; j.rf_nblk = ph.Npad; j.rf_steps = (int)ph.steps.size();
    j.rf_row16 = ph.CbG * ph.pslab16; j.rf_total_rows = ph.rf_R + KH - 1;
    j.nrows = ph.rf_rps; j.ngroups = j.rf_total_rows / ph.rf_rps;
    for (int g = 0; g < j.ngroups; ++g) {
      j.grp_cb0[g] = 0;
      for (int ri = 0; ri < j.nrows; ++ri) j.grp_row[g][ri] = in.padT + ph.rows[0] + g * ph.rf_rps + ri;
    }
  }
  j.pslab16 = ph.pslab16; j.stage16 = j.nrows * ph.CbG * ph.pslab16;
  j.nchunks = ph.nchunks; j.spc = ph.spc;
  for (size_t i = 0; i < ph.steps.size(); ++i) j.steps[i] = ph.steps[i];
  j.chunk16 = 2 * ph.spc * 2 * ph.Npad; j.Npad = ph.Npad; j.Cout = c.cout;
  if (ph.rf_R) { j.nchunks = j.rf_steps; j.spc = 1; j.chunk16 = 2 * 2 * j.rf_kh * ph.Npad; }  // one resident chunk per K step
  if (ph.pf) {
    j.pf = 1; j.pf_cout = c.cout; j.mt = 1;
    int src = 0;
    for (int t = 0; t < 4; ++t) {
      j.pf_n[t] = kPfNblk[t] * c.cout; j.pf_col[t] = kPfBlk0[t] * c.cout;
      j.pf_len16[t] = 2 * ph.spc * 2 * j.pf_n[t]; j.pf_src16[t] = src;
      src += j.pf_len16[t];
    }
    j.pf_grp16 = src;
    j.chunk16 = j.pf_len16[0];  // slot size = largest chunk (tap (0,0): all four phases)
    j.oy_mul = j.ox_mul = 2; j.oy_off = j.ox_off = 0;
  }
  j.ksplit = 0;
  if (ph.rf_R) {  // per-patch-row issue table (conv_tc.cu, row-fold loop)
    const int KH = j.rf_kh, R = j.rf_R, nblk = j.rf_nblk;
    if (j.rf_total_rows > kMaxRfRows) { set_error("conv %s: row-fold unit too tall", c.name.c_str()); return FAV_ERR_UNSUPPORTED; }
    const uint32_t idesc_base = (1u << 4) | ((uint32_t)(kTileM >> 4) << 24);
    auto idn = [&](int rows) { return rows > 0 ? idesc_base | ((uint32_t)((rows * nblk) >> 3) << 17) : 0u; };
    for (int iy = 0; iy < j.rf_total_rows; ++iy) {
      const int r_min = iy - (KH - 1) > 0 ? iy - (KH - 1) : 0, r_max = iy < R - 1 ? iy : R - 1;
      const int nb = r_max - r_min + 1, blk0 = KH - 1 - (iy - r_min);
      // rows this issuing warp touches for the first time: r = iy (ky = 0) and, K-split, r = iy - 1 as well
      const int nf = (iy < R ? 1 : 0) + ((j.ksplit && iy >= 1 && iy - 1 < R) ? 1 : 0);
      j.rf_dcol[iy] = (uint32_t)(r_min * nblk); j.rf_boff[iy] = (uint32_t)(blk0 * nblk);
      j.rf_idn_all[iy] = idn(nb); j.rf_idn_acc[iy] = idn(nb - nf); j.rf_idn_new[iy] = idn(nf);
      j.rf_off_new[iy] = (uint32_t)((nb - nf) * nblk);
    }
  }
  j.oy_mul = c.out_mul; j.ox_mul = c.out_mul; j.oy_off = ph.oy_off; j.ox_off = ph.ox_off;
  j.nstack = ph.nstack;
  for (int s = 0; s < ph.nstack; ++s) { j.st_oy[s] = ph.stack_oy[s]; j.st_ox[s] = ph.stack_ox[s]; }
  // every bulk copy must stay inside the operand allocation
  int64_t max_row = (int64_t)j.row_mul * (ceil_div(pHo, j.mt) * j.mt - 1) + in.padT + ph.rows.back();
  if (ph.rf_R) max_row = (int64_t)(ceil_div(pHo, j.mt) - 1) * j.mt + in.padT + ph.rows[0] + j.rf_total_rows - 1;
  int64_t last16 = ((max_row * in.Cb + in.Cb - 1) * (int64_t)in.slab16()) + j.seg_src16[ph.nseg - 1] +
                   (int64_t)(j.tiles_x - 1) * j.tile_dx + j.seg_len16[ph.nseg - 1];
  if (max_row >= in.Hs || last16 > (int64_t)in.elems16) {
    set_error("conv %s: internal operand bounds error", c.name.c_str());
    return FAV_ERR_INVALID;
  }
  return FAV_OK;
}

}  // namespace fav
