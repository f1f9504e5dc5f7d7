// conv_emu.cu -- TEST INFRASTRUCTURE: a CPU emulation of conv_tc_kernel's ADDRESSING (bulk-copy segments, patch
// stages, K-step tables, canonical no-swizzle K-major UMMA operand layout, packed weight chunks, output
// placement) driven by the very same host planning code the product uses (csrc/conv_plan.hpp).  It checks the
// tables against a direct convolution, so that table / packing bugs are caught here on the CPU and GPU time is
// spent on hardware semantics only.  Not part of libfav_b200.so.
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <random>
#include <vector>

#include "../../fast-artistic-videos_b200/csrc/conv_plan.hpp"

namespace fav {
static char g_err[512];
void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
std::atomic<uint64_t> g_launches{0};
// mirror of conv_tc.cu: kNA = 2 patch stages, up to 16 weight slots (resident when every chunk fits)
static size_t tc_fixed_smem(const ConvJob &job) {
  return (size_t)job.a_stages * 2 * job.stage16 * 16 + 640 + (job.xfold_kw ? (size_t)(job.mt >= 2 ? 2 : 1) * 128 * 33 * 4 : (size_t)(256 + 2048) * 4);
}
size_t conv_tc_smem_bytes(const ConvJob &job) { return tc_fixed_smem(job) + (size_t)job.b_slots * job.chunk16 * 16; }
void conv_tc_choose_slots(ConvJob &job) {
  const size_t budget = 224 * 1024, chunk = (size_t)job.chunk16 * 16;
  const int total = job.rf_R ? job.rf_steps : (job.pf ? job.ngroups * 4 : job.ngroups * job.nchunks);
  job.a_stages = 2;
  {
    ConvJob t = job;
    for (int n = 4; n > 2; --n) {
      t.a_stages = n;
      if (total <= 16 && tc_fixed_smem(t) + total * chunk <= budget) { job.a_stages = n; break; }
    }
  }
  const size_t fixed = tc_fixed_smem(job);
  if (total <= 16 && fixed + total * chunk <= budget) { job.b_resident = 1; job.b_slots = total; }
  else { job.b_resident = 0; int n = (int)((budget - fixed) / chunk); job.b_slots = n > 16 ? 16 : (n < 2 ? 2 : n); }
}
}  // namespace fav

using namespace fav;

extern "C" const char *emu_last_error() { return fav::g_err; }

// returns 0 on success; max_err = max |emulated - direct|, max_ref = max |direct|
extern "C" int emu_conv_check(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int H, int W,
                              unsigned seed, double *max_err, double *max_ref, int *smem_bytes, int *n_mma) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  std::vector<float> w((size_t)cin * cout * k * k), x((size_t)cin * H * W);
  for (auto &v : w) v = U(rng) * 0.1f;
  for (auto &v : x) v = U(rng) * 3.f;
  // operand (host mirror)
  Operand op = operand_geometry(cin, H, W, &c);
  std::vector<uint16_t> hi(op.elems16 * 8, 0), lo(op.elems16 * 8, 0);
  std::vector<float> xq((size_t)cin * H * W);
  for (int ci = 0; ci < cin; ++ci)
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float v = x[((size_t)ci * H + y) * W + xx];
        uint16_t hb = f2h_bits(v), lb = f2h_bits(v - h2f_bits(hb));
        int64_t o = op.off16(op.padT + y, ci / 8, op.padL + xx) * 8 + ci % 8;
        hi[o] = hb; lo[o] = lb;
        xq[((size_t)ci * H + y) * W + xx] = h2f_bits(hb) + h2f_bits(lb);
      }
  int Ho, Wo;
  conv_out_size(c, H, W, &Ho, &Wo);
  std::vector<double> out((size_t)cout * Ho * Wo, 0.0), ref((size_t)cout * Ho * Wo, 0.0);
  std::vector<char> written((size_t)Ho * Wo, 0);
  int mma_count = 0;
  size_t smem_max = 0;
  set_weight_prescale(c, w);
  std::vector<ConvPhase *> todo;
  if (c.has_fold) todo.push_back(&c.fold);
  else for (ConvPhase &p : c.phases) todo.push_back(&p);
  for (ConvPhase *php : todo) {
    ConvPhase &ph = *php;
    if (!ph.pf && build_phase_tables(c, ph) != FAV_OK) return 1;
    std::vector<uint16_t> pk = ph.pf ? pack_phase_fold(c, ph, w) : pack_phase_weights(c, ph, w);
    ConvJob j;
    if (fill_conv_job(c, ph, op, j) != FAV_OK) return 2;
    conv_tc_choose_slots(j);
    if (j.b_slots < 2 && !j.b_resident) { set_error("weight ring too small"); return 9; }
    smem_max = std::max(smem_max, conv_tc_smem_bytes(j));
    if (conv_tc_smem_bytes(j) > 227 * 1024) { set_error("smem budget"); return 3; }
    const int Npad = j.Npad;
    std::vector<uint16_t> st_hi((size_t)j.stage16 * 8), st_lo((size_t)j.stage16 * 8);
    std::vector<double> acc(j.rf_R ? (size_t)kTileM * 512 : (size_t)2 * kTileM * Npad);
    std::vector<double> acc2(acc.size());  // K-split: the second issuing warp's accumulator (columns +128)
    if (j.ksplit && (j.rf_R ? j.rf_R * j.rf_nblk : Npad) > 128) { set_error("ksplit needs <= 128 columns"); return 10; }
    if (j.ksplit && j.mt != 1 && !j.rf_R) { set_error("ksplit with mt = 2"); return 10; }
    for (int tile = 0; tile < j.ntiles; ++tile) {
      const int y = (tile / j.tiles_x) * j.mt, x0 = (tile % j.tiles_x) * j.tile_dx;
      const double poison = (j.rf_R || j.ksplit) ? 1e30 : 0.0;  // a stale accumulator must be overwritten, not accumulated
      std::fill(acc.begin(), acc.end(), poison);
      std::fill(acc2.begin(), acc2.end(), poison);
      bool first_w[2] = {true, true};  // K-split: first MMA of each issuing warp in the unit (accumulate = 0)
      int sc = 0;                       // K-step counter of the unit
      for (int g = 0; g < j.ngroups; ++g) {
        // A producer
        std::fill(st_hi.begin(), st_hi.end(), (uint16_t)0x7e00);  // NaN poison: reading an unloaded byte is a bug
        std::fill(st_lo.begin(), st_lo.end(), (uint16_t)0x7e00);
        for (int ri = 0; ri < j.nrows; ++ri)
          for (int cbi = 0; cbi < j.CbG; ++cbi)
            for (int seg = 0; seg < j.nseg; ++seg) {
              int64_t src16 = ((int64_t)(j.row_mul * y + j.grp_row[g][ri]) * j.a_Cb + j.grp_cb0[g] + cbi) * j.a_slab16 +
                              j.seg_src16[seg] + x0;
              int64_t dst16 = (int64_t)(ri * j.CbG + cbi) * j.pslab16 + j.seg_dst16[seg];
              if (src16 < 0 || src16 + j.seg_len16[seg] > (int64_t)op.elems16) { set_error("src OOB"); return 4; }
              if (dst16 + j.seg_len16[seg] > j.stage16) { set_error("dst OOB"); return 5; }
              for (int64_t e = 0; e < (int64_t)j.seg_len16[seg] * 8; ++e) {
                st_hi[dst16 * 8 + e] = hi[src16 * 8 + e];
                st_lo[dst16 * 8 + e] = lo[src16 * 8 + e];
              }
            }
        if (j.rf_R) {
          // row-fold: patch row iy -> output rows r_min..r_max, weights slice of the descending-ky image (conv.cuh)
          const int KH = j.rf_kh, R = j.rf_R, nblk = j.rf_nblk, NR = KH * nblk;
          for (int ri = 0; ri < j.nrows; ++ri) {
            const int iy = g * j.nrows + ri;
            std::vector<double> &accw = (j.ksplit && (iy & 1)) ? acc2 : acc;  // K-split: patch rows by parity
            const int nf = (iy < R ? 1 : 0) + ((j.ksplit && iy >= 1 && iy - 1 < R) ? 1 : 0);
            const int r_min = std::max(0, iy - (KH - 1)), r_max = std::min(R - 1, iy);
            const int nb = r_max - r_min + 1, blk0 = KH - 1 - (iy - r_min);
            {  // the kernel reads these from the host-computed per-row table
              const uint32_t ib = (1u << 4) | ((uint32_t)(kTileM >> 4) << 24);
              auto idn = [&](int rows) { return rows > 0 ? ib | ((uint32_t)((rows * nblk) >> 3) << 17) : 0u; };
              if (j.rf_dcol[iy] != (uint32_t)(r_min * nblk) || j.rf_boff[iy] != (uint32_t)(blk0 * nblk) ||
                  j.rf_idn_all[iy] != idn(nb) || j.rf_idn_acc[iy] != idn(nb - nf) || j.rf_idn_new[iy] != idn(nf) ||
                  j.rf_off_new[iy] != (uint32_t)((nb - nf) * nblk)) { set_error("row-fold table mismatch at row %d", iy); return 11; }
            }
            for (int st = 0; st < j.rf_steps; ++st) {
              const KStep ks = j.steps[st];
              const uint16_t *chunk = pk.data() + (size_t)st * j.chunk16 * 8;   // [hi: 2 x NR rows][lo: 2 x NR rows]
              const bool fresh = (st == 0 && nf > 0);
              mma_count += 3 * (fresh && nb > nf ? 2 : 1);
              for (int m = 0; m < kTileM; ++m)
                for (int u = 0; u < 2; ++u) {
                  int64_t a16 = (int64_t)ri * j.rf_row16 + ks.a_off16 + (int64_t)u * ks.lbo16 + m;
                  if (a16 >= j.stage16) { set_error("A desc OOB (rowfold)"); return 6; }
                  for (int i = 0; i < 8; ++i) {
                    double ah = h2f_bits(st_hi[a16 * 8 + i]), al = h2f_bits(st_lo[a16 * 8 + i]);
                    for (int n = 0; n < nb * nblk; ++n) {
                      int64_t brow = (int64_t)blk0 * nblk + n;              // row inside one k-half image
                      if (brow >= NR) { set_error("B desc OOB (rowfold)"); return 6; }
                      double bh = h2f_bits(chunk[((int64_t)u * NR + brow) * 8 + i]);
                      double bl = h2f_bits(chunk[((int64_t)(2 + u) * NR + brow) * 8 + i]);
                      size_t col = (size_t)r_min * nblk + n;               // accumulator column
                      double &d = accw[(size_t)m * 512 + col];
                      const bool overwrite = fresh && (n >= (nb - nf) * nblk) && u == 0 && i == 0;
                      if (overwrite) d = 0;                                  // accumulate = 0 on the first MMA of the new row
                      d += ah * bh + al * bh + ah * bl;
                    }
                  }
                }
            }
          }
          continue;
        }
        if (j.pf) {
          // phase-fold: chunk = tap; N = pf_n[ch] columns starting at pf_col[ch]
          for (int ch = 0; ch < 4; ++ch) {
            const int n_ = j.pf_n[ch];
            if (j.pf_len16[ch] > j.chunk16) { set_error("pf chunk larger than slot"); return 6; }
            const uint16_t *chunk = pk.data() + ((size_t)g * j.pf_grp16 + j.pf_src16[ch]) * 8;
            const uint16_t *b_hi = chunk, *b_lo = chunk + (size_t)j.spc * 2 * n_ * 8;
            for (int st = 0; st < j.spc; ++st) {
              const KStep ks = j.steps[ch * j.spc + st];
              mma_count += 3;
              const int w = j.ksplit ? (st & 1) : 0;
              std::vector<double> &accw = w ? acc2 : acc;
              if (j.ksplit && first_w[w]) {  // accumulate = 0: must cover every column
                if (j.pf_col[ch] != 0 || n_ != Npad) { set_error("pf ksplit: first MMA does not cover all columns"); return 6; }
                for (int m = 0; m < kTileM; ++m) for (int n = 0; n < n_; ++n) accw[(size_t)m * Npad + n] = 0;
                first_w[w] = false;
              }
              for (int m = 0; m < kTileM; ++m)
                for (int u = 0; u < 2; ++u) {
                  int64_t a16 = (int64_t)ks.a_off16 + (int64_t)u * ks.lbo16 + m;
                  if (a16 >= j.stage16) { set_error("A desc OOB (pf)"); return 6; }
                  for (int i = 0; i < 8; ++i) {
                    double ah = h2f_bits(st_hi[a16 * 8 + i]), al = h2f_bits(st_lo[a16 * 8 + i]);
                    for (int n = 0; n < n_; ++n) {
                      int64_t b16 = (int64_t)st * 2 * n_ + (int64_t)u * n_ + n;
                      if ((b16 + 1) > j.pf_len16[ch] / 2) { set_error("B desc OOB (pf)"); return 6; }
                      double bh = h2f_bits(b_hi[b16 * 8 + i]), bl = h2f_bits(b_lo[b16 * 8 + i]);
                      accw[(size_t)m * Npad + j.pf_col[ch] + n] += ah * bh + al * bh + ah * bl;
                    }
                  }
                }
            }
          }
          continue;
        }
        for (int ch = 0; ch < j.nchunks; ++ch) {
          const uint16_t *chunk = pk.data() + (size_t)(g * j.nchunks + ch) * j.chunk16 * 8;
          const uint16_t *b_hi = chunk, *b_lo = chunk + (size_t)j.spc * 2 * Npad * 8;
          for (int st = 0; st < j.spc; ++st) {
            const KStep ks = j.steps[ch * j.spc + st];
            mma_count += 3 * j.mt;
            const int w = j.ksplit ? ((sc + st) & 1) : 0;
            std::vector<double> &accw = w ? acc2 : acc;
            if (j.ksplit && first_w[w]) { std::fill(accw.begin(), accw.end(), 0.0); first_w[w] = false; }
            for (int t = 0; t < j.mt; ++t)
            for (int m = 0; m < kTileM; ++m)
              for (int u = 0; u < 2; ++u) {
                // row m: +16 B (SBO = 8 rows * 16 B); second output row of an mt=2 unit: one patch row lower
                int64_t a16 = (int64_t)ks.a_off16 + (int64_t)u * ks.lbo16 + m + (int64_t)t * j.CbG * j.pslab16;
                if (a16 >= j.stage16) { set_error("A desc OOB"); return 6; }
                for (int i = 0; i < 8; ++i) {
                  double ah = h2f_bits(st_hi[a16 * 8 + i]), al = h2f_bits(st_lo[a16 * 8 + i]);
                  for (int n = 0; n < Npad; ++n) {
                    int64_t b16 = (int64_t)st * 2 * Npad + (int64_t)u * Npad + n;
                    double bh = h2f_bits(b_hi[b16 * 8 + i]), bl = h2f_bits(b_lo[b16 * 8 + i]);
                    accw[((size_t)t * kTileM + m) * Npad + n] += ah * bh + al * bh + ah * bl;
                  }
                }
              }
          }
          sc += j.spc;
        }
      }
      // epilogue: K-split units add the second warp's accumulator
      if (j.ksplit)
        for (size_t i = 0; i < acc.size(); ++i) acc[i] += acc2[i];
      for (double &v : acc) v *= j.w_unscale;  // the packed weights are w * 2^w_exp
      // epilogue placement
      if (j.rf_R) {
        const int nblk = j.rf_nblk;
        for (int t = 0; t < j.rf_R; ++t)
          for (int m = 0; m < (j.xfold_kw ? j.tile_dx : kTileM); ++m) {
            int xx = x0 + m;
            if (xx >= j.Wo || y + t >= j.Ho) continue;
            written[(size_t)(y + t) * Wo + xx]++;
            for (int n = 0; n < cout; ++n) {
              double v = 0;
              if (j.xfold_kw) for (int kx = 0; kx < j.xfold_kw; ++kx) v += acc[(size_t)(m + kx) * 512 + (size_t)t * nblk + kx * cout + n];
              else v = acc[(size_t)m * 512 + (size_t)t * nblk + n];
              out[((size_t)n * Ho + y + t) * Wo + xx] = v;
            }
          }
        continue;
      }
      if (j.pf) {
        for (int m = 0; m < kTileM; ++m) {
          int xx = x0 + m;
          if (xx >= j.Wo || y >= j.Ho) continue;
          for (int blk = 0; blk < 4; ++blk) {
            const int a = blk >> 1, b = (blk == 1 || blk == 2) ? 1 : 0;
            int yo = 2 * y + a, xo = 2 * xx + b;
            if (yo >= Ho || xo >= Wo) { set_error("output OOB (pf)"); return 7; }
            written[(size_t)yo * Wo + xo]++;
            for (int n = 0; n < cout; ++n) out[((size_t)n * Ho + yo) * Wo + xo] = acc[(size_t)m * Npad + blk * j.pf_cout + n];
          }
        }
        continue;
      }
      if (j.xfold_kw) {
        for (int m = 0; m < j.tile_dx; ++m) {
          int xx = x0 + m;
          if (xx >= j.Wo) continue;
          written[(size_t)y * Wo + xx]++;
          for (int n = 0; n < cout; ++n) {
            double sacc = 0;
            for (int kx = 0; kx < j.xfold_kw; ++kx) sacc += acc[(size_t)(m + kx) * Npad + kx * cout + n];
            out[((size_t)n * Ho + y) * Wo + xx] = sacc;
          }
        }
        continue;
      }
      for (int t = 0; t < j.mt; ++t)
      for (int m = 0; m < kTileM; ++m) {
        int xx = x0 + m;
        if (xx >= j.Wo || y + t >= j.Ho) continue;
        int yo = (y + t) * j.oy_mul + j.oy_off, xo = xx * j.ox_mul + j.ox_off;
        if (yo >= Ho || xo >= Wo) { set_error("output OOB"); return 7; }
        written[(size_t)yo * Wo + xo]++;
        for (int n = 0; n < cout; ++n) out[((size_t)n * Ho + yo) * Wo + xo] = acc[((size_t)t * kTileM + m) * Npad + n];
      }
    }
  }
  for (char wv : written)
    if (wv != 1) { set_error("output pixel written %d times", (int)wv); return 8; }
  // direct reference
  if (!transposed) {
    for (int co = 0; co < cout; ++co)
      for (int oy = 0; oy < Ho; ++oy)
        for (int ox = 0; ox < Wo; ++ox) {
          double s = 0;
          for (int ci = 0; ci < cin; ++ci)
            for (int ky = 0; ky < k; ++ky) {
              int iy = oy * stride + ky - pad;
              if (iy < 0 || iy >= H) continue;
              for (int kx = 0; kx < k; ++kx) {
                int ix = ox * stride + kx - pad;
                if (ix < 0 || ix >= W) continue;
                s += (double)w[(((size_t)co * cin + ci) * k + ky) * k + kx] * xq[((size_t)ci * H + iy) * W + ix];
              }
            }
          ref[((size_t)co * Ho + oy) * Wo + ox] = s;
        }
  } else {
    for (int ci = 0; ci < cin; ++ci)
      for (int iy = 0; iy < H; ++iy)
        for (int ix = 0; ix < W; ++ix) {
          double xv = xq[((size_t)ci * H + iy) * W + ix];
          for (int ky = 0; ky < k; ++ky) {
            int oy = iy * stride - pad + ky;
            if (oy < 0 || oy >= Ho) continue;
            for (int kx = 0; kx < k; ++kx) {
              int ox = ix * stride - pad + kx;
              if (ox < 0 || ox >= Wo) continue;
              for (int co = 0; co < cout; ++co)
                ref[((size_t)co * Ho + oy) * Wo + ox] += xv * w[(((size_t)ci * cout + co) * k + ky) * k + kx];
            }
          }
        }
  }
  double me = 0, mr = 0;
  for (size_t i = 0; i < ref.size(); ++i) {
    double d = std::fabs(out[i] - ref[i]);
    if (!(d <= 1e300)) d = 1e300;  // NaN -> huge
    me = std::max(me, d);
    mr = std::max(mr, std::fabs(ref[i]));
  }
  *max_err = me; *max_ref = mr;
  if (smem_bytes) *smem_bytes = (int)smem_max;
  if (n_mma) *n_mma = mma_count;
  return 0;
}

// planner decisions for one layer (first job): {mt, ksplit, pf, rf_R, xfold_kw, b_resident, a_stages, b_slots, ntiles, Npad}
extern "C" int emu_plan_info(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int H, int W, int *out10) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  Operand op = operand_geometry(cin, H, W, &c);
  ConvPhase &ph = c.has_fold ? c.fold : c.phases[0];
  if (!ph.pf && build_phase_tables(c, ph) != FAV_OK) return 1;
  ConvJob j;
  if (fill_conv_job(c, ph, op, j) != FAV_OK) return 2;
  conv_tc_choose_slots(j);
  const int v[10] = {j.mt, j.ksplit, j.pf, j.rf_R, j.xfold_kw, j.b_resident, j.a_stages, j.b_slots, j.ntiles, j.Npad};
  for (int i = 0; i < 10; ++i) out10[i] = v[i];
  return 0;
}


extern "C" int emu_plan_detail(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int H, int W, int *out16) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  Operand op = operand_geometry(cin, H, W, &c);
  ConvPhase &ph = c.has_fold ? c.fold : c.phases[0];
  if (!ph.pf && build_phase_tables(c, ph) != FAV_OK) return 1;
  ConvJob j;
  if (fill_conv_job(c, ph, op, j) != FAV_OK) return 2;
  conv_tc_choose_slots(j);
  const int v[16] = {j.ngroups, j.nchunks, j.spc, j.nrows, j.CbG, j.nseg, j.a_stages, j.b_slots, j.b_resident, j.stage16 * 16,
                     j.chunk16 * 16, j.pslab16, j.tiles_x, j.ntiles, j.Npad, j.ksplit};
  for (int i = 0; i < 16; ++i) out16[i] = v[i];
  return 0;
}

// ---- weight prescale (set_weight_prescale, weight_half): every packing path against the weights it packs -----------------
// A packed job does not say which weight each of its fp16 pairs holds, so the job is packed twice: once from the weights and
// once from their indices (index i + 1 as the weight value; max < 2^22, so hi + lo holds it exactly).  Position p then holds
// weight idx[p] and must decode, as hi + lo times the job's 2^-w_exp, to within 2^-21 of it: relative to the weight itself, or to
// the pair's floor 2^-4 in packed units (2^-4-e in weight units): lo's subnormal step 2^-24 bounds the error by 2^-25.
struct PackedJob {
  ConvDef c;            // the ConvDef the job is packed from (an N block, or the whole convolution)
  const ConvPhase *ph;  // the phase (tables) it packs
  std::vector<float> w, idx;
  int path;             // 0: pack_phase_weights, 1: row-fold image, 2: pack_phase_fold
  int e;                // the exponent the job runs with: ConvJob::w_unscale = 2^-e (row-fold: ConvDef::w_exp)
};

// distance (uint16 elements) from each hi element to its lo partner, and whether element p is a hi element
static bool hi_element(const PackedJob &pj, size_t p, size_t *lo_off) {
  const ConvPhase &ph = *pj.ph;
  if (pj.path == 1) {  // [step][hi|lo][k-half][NR][8]
    const size_t B = (size_t)2 * ph.rows.size() * ph.Npad * 8;
    *lo_off = B;
    return (p / B) % 2 == 0;
  }
  if (pj.path == 2) {  // [group][tap chunk: [hi|lo][spc][k-half][n][8]]
    const int spc = ph.CbG / 2;
    size_t grp = 0;
    for (int t = 0; t < 4; ++t) grp += (size_t)2 * spc * 2 * kPfNblk[t] * pj.c.cout * 8;
    size_t q = p % grp;
    for (int t = 0; t < 4; ++t) {
      const size_t B = (size_t)spc * 2 * kPfNblk[t] * pj.c.cout * 8;
      if (q < 2 * B) { *lo_off = B; return q < B; }
      q -= 2 * B;
    }
    return false;
  }
  const size_t B = (size_t)ph.spc * 2 * ph.Npad * 8;  // [group][chunk][hi|lo][step][k-half][Npad][8]
  *lo_off = B;
  return (p / B) % 2 == 0;
}

static std::vector<uint16_t> pack_job(const PackedJob &pj, const ConvDef &c, const std::vector<float> &w) {
  return pj.path == 2 ? pack_phase_fold(c, *pj.ph, w) : pack_phase_weights(c, *pj.ph, w);
}

// the row-fold tables build_phase_tables gives a tap-paired (kind 1) or x-fold (kind 3) phase when kPlanRowFold is on: the K
// steps of one patch row, all channel blocks in one stage
static void rowfold_tables(const ConvDef &c, ConvPhase &ph) {
  ph.steps.clear();
  ph.units.assign(1, {});
  if (ph.kind == 1) {
    const int ndx = ph.dxmax - ph.dxmin + 1;
    for (int p = 0; p * 2 < ndx; ++p) {
      ph.steps.push_back(KStep{(uint16_t)(2 * p), 1});
      for (int u = 0; u < 2; ++u) ph.units[0].push_back(Unit{2 * p + u < ndx ? 2 * p + u : -1, 0});
    }
  } else {
    ph.CbG = c.Cb; ph.nchg = 1;
    for (int j = 0; j < ph.CbG / 2; ++j) {
      ph.steps.push_back(KStep{(uint16_t)(2 * j * ph.pslab16), (uint16_t)ph.pslab16});
      for (int u = 0; u < 2; ++u) ph.units[0].push_back(Unit{0, 2 * j + u});
    }
  }
  ph.rf_R = 4; ph.nrg = 1; ph.spc = (int)ph.steps.size(); ph.nchunks = 1;
}

// path 0: every job the stylization net / loss network packs for the convolution (N blocks x sub-pixel phases, stacked phases,
// x-fold when !raw_out); 1: the row-fold image of its first phase (tap-paired or x-fold); 2: the phase-fold job (f3s2).
// Weights U(-1, 1)^3 * wscale (0: all zero).  out: [0] worst error / bound, [1] max |w| 2^e, [2] jobs, [3] distinct exponents,
// [4] weights no job packs.  *e_out: the exponent of the first job.
extern "C" int emu_weight_scale_check(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int raw_out, int path,
                                      double wscale, unsigned seed, double *out, int *e_out) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  c.raw_out = raw_out != 0;
  std::mt19937 rng(seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::vector<float> w((size_t)cin * cout * k * k), idx(w.size());
  double maxw = 0;
  for (size_t i = 0; i < w.size(); ++i) {
    const double u = U(rng);
    w[i] = (float)(u * u * u * wscale);
    if (i == 0) w[i] = (float)(0.999 * wscale);  // one weight near the top of the binade
    idx[i] = (float)(i + 1);
    maxw = std::max(maxw, (double)std::fabs(w[i]));
  }
  if (idx.size() >= (1u << 22)) { set_error("too many weights to index exactly"); return 1; }
  Operand op = operand_geometry(cin, 16, 16, &c);
  std::vector<PackedJob> jobs;
  std::vector<ConvPhase> extra;  // row-fold / phase-fold tables
  extra.reserve(1);
  if (path == 0) {
    if (plan_conv_nblocks(c) != FAV_OK || plan_phase_stack(c) != FAV_OK) return 2;
    set_weight_prescale(c, w);
    if (!c.nblock.empty()) {
      for (int b = 0; b < (int)c.nblock.size(); ++b)
        for (const ConvPhase &ph : c.nblock[b].phases)
          jobs.push_back(PackedJob{c.nblock[b], &ph, conv_nblock_weights(w, cin, cout, k, b, c.transposed),
                                   conv_nblock_weights(idx, cin, cout, k, b, c.transposed), 0, 0});
    } else {
      for (const ConvPhase &ph : c.phases) jobs.push_back(PackedJob{c, &ph, w, idx, 0, 0});
    }
    for (const ConvPhase &ph : c.stack) jobs.push_back(PackedJob{c, &ph, w, idx, 0, 0});
  } else if (path == 1) {
    extra.push_back(c.phases[0]);
    if (build_phase_tables(c, extra[0]) != FAV_OK) return 2;
    if (extra[0].kind != 1 && extra[0].kind != 3) { set_error("row-fold needs a tap-paired or x-fold phase, got kind %d", extra[0].kind); return 3; }
    rowfold_tables(c, extra[0]);
    set_weight_prescale(c, w);
    jobs.push_back(PackedJob{c, &extra[0], w, idx, 1, 0});
  } else {
    extra.push_back(ConvPhase());
    if (build_phase_fold(c, extra[0]) != FAV_OK) { set_error("no phase-fold plan"); return 3; }
    set_weight_prescale(c, w);
    jobs.push_back(PackedJob{c, &extra[0], w, idx, 2, 0});
  }
  std::vector<int> seen(w.size(), 0), exps;
  double worst = 0;
  for (PackedJob &pj : jobs) {
    if (pj.path == 1) {
      pj.e = pj.c.w_exp;
    } else {
      ConvJob j;
      if (fill_conv_job(pj.c, *pj.ph, op, j) != FAV_OK) return 4;
      pj.e = -ilogbf(j.w_unscale);
      if (j.w_unscale != ldexpf(1.f, -pj.e)) { set_error("w_unscale %g is not a power of two", j.w_unscale); return 5; }
    }
    if (std::find(exps.begin(), exps.end(), pj.e) == exps.end()) exps.push_back(pj.e);
    const std::vector<uint16_t> pw = pack_job(pj, pj.c, pj.w);
    ConvDef ci = pj.c;
    ci.w_exp = weight_prescale_exp(pj.idx);
    const std::vector<uint16_t> pi = pack_job(pj, ci, pj.idx);
    if (pw.size() != pi.size()) { set_error("packed sizes differ"); return 6; }
    for (size_t p = 0; p < pw.size(); ++p) {
      size_t lo_off = 0;
      if (!hi_element(pj, p, &lo_off)) continue;
      if (p + lo_off >= pw.size()) { set_error("lo element out of range"); return 7; }
      const double id = ldexp((double)h2f_bits(pi[p]) + h2f_bits(pi[p + lo_off]), -ci.w_exp);
      const double got = ldexp((double)h2f_bits(pw[p]) + h2f_bits(pw[p + lo_off]), -pj.e);
      if (id == 0) {  // a zero tap or padding
        if (pw[p] != 0 || pw[p + lo_off] != 0) { set_error("padding element %zu holds %g", p, got); return 8; }
        continue;
      }
      const long long i = std::llround(id) - 1;
      if (i < 0 || i >= (long long)w.size() || (double)(i + 1) != id) { set_error("element %zu decodes to index %g", p, id); return 9; }
      seen[i]++;
      const double ref = w[i], err = std::fabs(got - ref);
      const double bound = std::ldexp(std::max(std::fabs(ref), std::ldexp(1.0, -4 - pj.e)), -21);
      const double r = bound > 0 ? err / bound : (err > 0 ? 1e300 : 0.0);
      if (!(r <= worst)) worst = std::isnan(r) ? 1e300 : r;
    }
  }
  int unseen = 0;
  for (int s : seen) unseen += s == 0;
  out[0] = worst; out[1] = std::ldexp(maxw, jobs[0].e); out[2] = (double)jobs.size(); out[3] = (double)exps.size();
  out[4] = unseen;
  *e_out = jobs[0].e;
  return 0;
}
