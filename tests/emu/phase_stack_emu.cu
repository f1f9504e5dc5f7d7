// phase_stack_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of conv_tc_kernel running the stacked sub-pixel phase jobs of a
// stride-2 transposed convolution (plan_phase_stack in conv_plan.hpp).  The jobs, tables, packed weights and bias come from the
// product's planner (plan_phase_stack, pack_phase_weights, stack_bias, fill_conv_job); the epilogue's output placement and
// statistics channel from the helpers the kernel calls (stack_epi_addr, stats_columns, stats_channel).  Not part of libfav_b200.so.
#include "nl_geom_emu.cu"

namespace {
ConvDef stacked_def(int cin, int cout, int k) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, 2, (k - 1) / 2, true, 1);  // fXs2-Z: SpatialFullConvolution(k, k, 2, 2, p, p, 1, 1)
  c.raw_out = true;
  build_phases(c);
  return c;
}
}  // namespace

// planner decisions: info[0] = stacked jobs (0: one job per phase), then per job {Npad, nstack, taps, b_resident} (up to 2 jobs)
extern "C" int emu_stack_plan(int cin, int cout, int k, int H, int W, int *info9) {
  ConvDef c = stacked_def(cin, cout, k);
  if (plan_conv_nblocks(c) != FAV_OK || plan_phase_stack(c) != FAV_OK) return 1;
  for (int i = 0; i < 9; ++i) info9[i] = 0;
  info9[0] = (int)c.stack.size();
  Operand op = operand_geometry(cin, H, W, &c);
  for (size_t s = 0; s < c.stack.size() && s < 2; ++s) {
    ConvJob j;
    if (fill_conv_job(c, c.stack[s], op, j) != FAV_OK) return 2;
    conv_tc_choose_slots(j);
    int *o = info9 + 1 + 4 * s;
    o[0] = j.Npad; o[1] = j.nstack; o[2] = (int)c.stack[s].taps.size(); o[3] = j.b_resident;
  }
  return 0;
}

// Every stacked job of fXs2-cout from cin channels on an H x W input, emulated tile by tile: patch staging from the job's
// tables, the packed hi / lo weights with the 3-MMA scheme (hi*hi + lo*hi + hi*lo), then the stacked epilogue of each of the
// 256 consumer threads (stack_epi_addr, stats_channel) into a raw [Ho][Cq][Wp][4] tensor and per-channel statistics.  Compared with a direct
// transposed convolution of the same fp16 hi + lo operand: max_err / max_ref of the outputs, stat_err = max relative error of
// the per-channel sums and sums of squares.  Every output element must be written exactly once.
extern "C" int emu_stack_check(int cin, int cout, int k, int H, int W, unsigned seed, double *max_err, double *max_ref,
                               double *stat_err) {
  ConvDef c = stacked_def(cin, cout, k);
  if (plan_conv_nblocks(c) != FAV_OK || plan_phase_stack(c) != FAV_OK) return 1;
  if (c.stack.empty()) { set_error("conv not stacked"); return 2; }
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  std::vector<float> w((size_t)cin * cout * k * k), x((size_t)cin * H * W), bias(cout);
  for (auto &v : w) v = U(rng) * 0.1f;
  for (auto &v : x) v = U(rng) * 3.f;
  for (auto &v : bias) v = U(rng);
  Operand op = operand_geometry(cin, H, W, &c);
  std::vector<uint16_t> hi(op.elems16 * 8, 0), lo(op.elems16 * 8, 0);
  std::vector<double> xq((size_t)cin * H * W);
  for (int ci = 0; ci < cin; ++ci)
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        const float v = x[((size_t)ci * H + y) * W + xx];
        const uint16_t hb = f2h_bits(v), lb = f2h_bits(v - h2f_bits(hb));
        const int64_t o = op.off16(op.padT + y, ci / 8, op.padL + xx) * 8 + ci % 8;
        hi[o] = hb; lo[o] = lb;
        xq[((size_t)ci * H + y) * W + xx] = (double)h2f_bits(hb) + h2f_bits(lb);
      }
  int Ho, Wo;
  conv_out_size(c, H, W, &Ho, &Wo);
  const int Cq = round_up(cout, 4) / 4, Wp = round_up(Wo, kTileM);
  std::vector<double> raw((size_t)Ho * Cq * Wp * 4, 0.0), ssum(cout, 0.0), ssq(cout, 0.0);
  std::vector<int> written(raw.size(), 0);
  const std::vector<float> sb = stack_bias(c, bias);
  set_weight_prescale(c, w);
  for (const ConvPhase &ph : c.stack) {
    const std::vector<uint16_t> pk = pack_phase_weights(c, ph, w);
    ConvJob j;
    if (fill_conv_job(c, ph, op, j) != FAV_OK) return 3;
    j.raw_Cq = Cq; j.raw_Wp = Wp;
    conv_tc_choose_slots(j);
    if (conv_tc_smem_bytes(j) > 227 * 1024 || (!j.b_resident && j.b_slots < 2)) { set_error("shared memory budget"); return 4; }
    if (j.nstack != ph.nstack || j.Npad > kMaxNBlock || j.Npad < j.nstack * j.Cout) { set_error("bad stacked job"); return 5; }
    const int Npad = j.Npad;
    std::vector<uint16_t> st_hi((size_t)j.stage16 * 8), st_lo((size_t)j.stage16 * 8);
    std::vector<double> acc((size_t)kTileM * Npad);
    std::vector<double> col_sum(Npad, 0.0), col_sq(Npad, 0.0);
    for (int T = 0; T < j.ntiles; ++T) {
      const TileAt at = tile_at(j, T);
      std::fill(acc.begin(), acc.end(), 0.0);
      for (int g = 0; g < j.ngroups; ++g) {
        std::fill(st_hi.begin(), st_hi.end(), (uint16_t)0x7e00);  // NaN poison: an unloaded byte must never be read
        std::fill(st_lo.begin(), st_lo.end(), (uint16_t)0x7e00);
        for (int ri = 0; ri < j.nrows; ++ri)
          for (int cbi = 0; cbi < j.CbG; ++cbi) {
            const int64_t src16 = ((int64_t)(j.row_mul * at.y + j.grp_row[g][ri]) * j.a_Cb + j.grp_cb0[g] + cbi) * j.a_slab16 +
                                  j.seg_src16[0] + at.x0;
            const int64_t dst16 = (int64_t)(ri * j.CbG + cbi) * j.pslab16 + j.seg_dst16[0];
            if (j.nseg != 1 || src16 < 0 || src16 + j.seg_len16[0] > (int64_t)op.elems16 || dst16 + j.seg_len16[0] > j.stage16) {
              set_error("patch copy out of bounds"); return 6;
            }
            for (int64_t e = 0; e < (int64_t)j.seg_len16[0] * 8; ++e) {
              st_hi[dst16 * 8 + e] = hi[src16 * 8 + e];
              st_lo[dst16 * 8 + e] = lo[src16 * 8 + e];
            }
          }
        for (int ch = 0; ch < j.nchunks; ++ch) {
          const uint16_t *chunk = pk.data() + (size_t)(g * j.nchunks + ch) * j.chunk16 * 8;
          const uint16_t *b_hi = chunk, *b_lo = chunk + (size_t)j.spc * 2 * Npad * 8;
          for (int st = 0; st < j.spc; ++st) {
            const KStep ks = j.steps[ch * j.spc + st];
            for (int m = 0; m < kTileM; ++m)
              for (int u = 0; u < 2; ++u) {
                const int64_t a16 = (int64_t)ks.a_off16 + (int64_t)u * ks.lbo16 + m;
                if (a16 >= j.stage16) { set_error("A descriptor out of the stage"); return 7; }
                for (int i = 0; i < 8; ++i) {
                  const double ah = h2f_bits(st_hi[a16 * 8 + i]), al = h2f_bits(st_lo[a16 * 8 + i]);
                  for (int n = 0; n < Npad; ++n) {
                    const int64_t b16 = (int64_t)st * 2 * Npad + (int64_t)u * Npad + n;
                    const double bh = h2f_bits(b_hi[b16 * 8 + i]), bl = h2f_bits(b_lo[b16 * 8 + i]);
                    acc[(size_t)m * Npad + n] += ah * bh + al * bh + ah * bl;
                  }
                }
              }
          }
        }
      }
      // the stacked epilogue of consumer thread t: accumulator rows r0, r0 + 8, column pairs 8i + 2 (t % 4); the statistics
      // stay per accumulator column until the flush below
      for (int t = 0; t < 256; ++t) {
        const int r0 = (t >> 7) * 64 + ((t >> 5) & 3) * 16 + ((t & 31) >> 2);
        for (int i = 0; i < Npad / 8; ++i)
          for (int h = 0; h < 2; ++h) {
            int64_t o = -1;
            if (!stack_epi_addr(j, at.y, at.x0, t, i, h, o)) continue;
            if (o < 0 || o + 1 >= (int64_t)raw.size()) { set_error("epilogue address out of range"); return 8; }
            for (int e = 0; e < 2; ++e) {
              const int n = 8 * i + 2 * (t & 3) + e;
              const double v = acc[(size_t)(r0 + 8 * h) * Npad + n] * j.w_unscale + sb[n];
              raw[o + e] = v;
              written[o + e]++;
              col_sum[n] += v;
              col_sq[n] += v * v;
            }
          }
      }
    }
    // tc_flush_stats: column n of the job into channel stats_channel(n)
    for (int n = 0; n < stats_columns(j); ++n) {
      const int ch = stats_channel(j, n);
      if (ch < 0 || ch >= cout) { set_error("statistics channel %d of column %d", ch, n); return 8; }
      ssum[ch] += col_sum[n];
      ssq[ch] += col_sq[n];
    }
  }
  // direct transposed convolution: out[oy = 2 iy - pad + ky][ox = 2 ix - pad + kx] += x[iy][ix] w[ci][co][ky][kx]
  std::vector<double> ref((size_t)cout * Ho * Wo);
  for (int co = 0; co < cout; ++co)
    for (size_t p = 0; p < (size_t)Ho * Wo; ++p) ref[(size_t)co * Ho * Wo + p] = bias[co];
  for (int ci = 0; ci < cin; ++ci)
    for (int iy = 0; iy < H; ++iy)
      for (int ix = 0; ix < W; ++ix) {
        const double xv = xq[((size_t)ci * H + iy) * W + ix];
        for (int ky = 0; ky < k; ++ky) {
          const int oy = 2 * iy - c.pad + ky;
          if (oy < 0 || oy >= Ho) continue;
          for (int kx = 0; kx < k; ++kx) {
            const int ox = 2 * ix - c.pad + kx;
            if (ox < 0 || ox >= Wo) continue;
            for (int co = 0; co < cout; ++co)
              ref[((size_t)co * Ho + oy) * Wo + ox] += xv * w[(((size_t)ci * cout + co) * k + ky) * k + kx];
          }
        }
      }
  double me = 0, mr = 0, se = 0;
  for (int co = 0; co < cout; ++co) {
    double rs = 0, rq = 0, ra = 0;
    for (int oy = 0; oy < Ho; ++oy)
      for (int ox = 0; ox < Wo; ++ox) {
        const size_t o = (((size_t)oy * Cq + co / 4) * Wp + ox) * 4 + co % 4;
        if (written[o] != 1) { set_error("output (%d, %d, %d) written %d times", co, oy, ox, written[o]); return 9; }
        const double r = ref[((size_t)co * Ho + oy) * Wo + ox];
        double d = std::fabs(raw[o] - r);
        if (!(d <= 1e300)) d = 1e300;
        me = std::max(me, d); mr = std::max(mr, std::fabs(r));
        rs += r; rq += r * r; ra += std::fabs(r);
      }
    se = std::max(se, std::fabs(ssum[co] - rs) / std::max(1.0, ra));
    se = std::max(se, std::fabs(ssq[co] - rq) / std::max(1.0, rq));
  }
  *max_err = me; *max_ref = mr; *stat_err = se;
  return 0;
}

// Norm-on-load of a stacked job (the method of emu_nl_geometry_check): fXs2-cout from cin channels reading the raw output of the
// previous conv ([B][H][Cq][Wp][4], junk past column W) through the norm-on-load producers.  For every (image, tile, group, patch
// row, channel block, pixel) of every stacked job, the stage the producers fill (nl_raw_row / nl_raw_col) must equal, hi and lo,
// byte for byte, the stage the bulk copies fill from the operand in_apply writes, except for pixels past the end of their slab
// (zero, outside the image, read by no stored output).  info[3]: stacked jobs, compared pixels, pixels past a slab end.
extern "C" int emu_stack_nl_check(int cin, int cout, int k, int H, int W, int B, unsigned seed, int *info) {
  ConvDef c = stacked_def(cin, cout, k);
  if (plan_conv_nblocks(c) != FAV_OK || plan_phase_stack(c) != FAV_OK) return 1;
  if (c.stack.empty()) { set_error("conv not stacked"); return 2; }
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-3.f, 3.f);
  for (int i = 0; i < 3; ++i) info[i] = 0;
  Raw prev;
  prev.t.C = cin; prev.t.Cq = round_up(cin, 4) / 4; prev.t.H = H; prev.t.W = W; prev.t.Hp = H + 2; prev.t.Wp = round_up(W, kTileM);
  prev.t.img = (int64_t)prev.t.Hp * prev.t.Cq * prev.t.Wp * 4 + 1024;
  prev.v.assign((size_t)(B * prev.t.img), 0.f);
  for (float &v : prev.v) v = U(rng);
  Operand cur = operand_geometry(cin, H, W, &c);
  cur.img16 = (int64_t)cur.elems16;
  Norm nm;
  nm.C = cin;
  for (int i = 0; i < B * cin; ++i) {
    nm.mean.push_back(U(rng) * 0.3f);
    nm.scale.push_back(0.2f + std::fabs(U(rng)));
    nm.beta.push_back(U(rng) * 0.5f);
  }
  const int64_t cells = (int64_t)B * cur.img16;
  std::vector<uint16_t> ohi((size_t)cells * 8, 0), olo((size_t)cells * 8, 0);
  for (int b = 0; b < B; ++b)
    for (int y = 0; y < H; ++y)
      for (int cb = 0; cb < cur.Cb; ++cb)
        for (int x = 0; x < W; ++x) {
          float v[8];
          for (int i = 0; i < 8; ++i) v[i] = prev.v[b * prev.t.img + prev.t.off4(y, 2 * cb + i / 4, x) * 4 + i % 4];
          const int64_t o = (b * cur.img16 + cur.off16(cur.padT + y, cb, cur.padL + x)) * 8;
          nm.apply(v, b, cb, &ohi[o], &olo[o]);
        }
  for (const ConvPhase &ph : c.stack) {
    ConvJob j;
    if (fill_conv_job(c, ph, cur, j) != FAV_OK) return 3;
    set_conv_batch(j, B, 0, 0, 0);
    set_norm_on_load(j, prev.t, cur, 1, nullptr, 2 * cin, nullptr, nullptr);
    if (!nl_geometry_ok(j)) { set_error("stacked job: no norm-on-load geometry"); return 4; }
    ++info[0];
    for (int T = 0; T < B * j.ntiles; ++T) {
      const TileAt at = tile_at(j, T);
      const int nvalid = std::min(j.tile_dx, j.Wo - at.x0);
      for (int g = 0; g < j.ngroups; ++g)
        for (int ri = 0; ri < j.nrows; ++ri)
          for (int cbi = 0; cbi < j.CbG; ++cbi) {
            const int cb = j.grp_cb0[g] + cbi, ry = nl_raw_row(j, at.y, g, ri);
            const int64_t srow = ((int64_t)(j.row_mul * at.y + j.grp_row[g][ri]) * j.a_Cb + cb) * j.a_slab16;
            for (int p = 0; p < j.pslab16; ++p) {
              const int scol = j.seg_src16[0] + at.x0 + p;
              const int64_t s16 = srow + scol + at.a16;
              if (s16 < 0 || s16 >= cells) { set_error("bulk source outside the operand (tile %d, pixel %d)", T, p); return 5; }
              uint16_t h8[8] = {0}, l8[8] = {0};
              const int x = nl_raw_col(j, at.x0, p);
              if (ry >= 0 && ry < j.nl_H && x >= 0 && x < j.nl_W) {
                float v[8];
                for (int i = 0; i < 8; ++i)
                  v[i] = prev.v[at.nl_raw4 * 4 + (((int64_t)ry * j.nl_Cq + 2 * cb + i / 4) * j.nl_Wp + x) * 4 + i % 4];
                nm.apply(v, at.b, cb, h8, l8);
              }
              ++info[1];
              if (!memcmp(h8, &ohi[s16 * 8], 16) && !memcmp(l8, &olo[s16 * 8], 16)) continue;
              bool zero = true;
              for (int i = 0; i < 8; ++i) zero = zero && !h8[i] && !l8[i];
              if (scol >= j.a_slab16 && zero && (x < 0 || x >= j.nl_W) && p > nvalid - 1 + j.pslab16 - kTileM) { ++info[2]; continue; }
              set_error("stage differs (tile %d, group %d, row %d, cb %d, pixel %d)", T, g, ri, cb, p);
              return 6;
            }
          }
    }
  }
  return 0;
}
