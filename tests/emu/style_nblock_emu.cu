// style_nblock_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of the stylization net's convolutions with more than 128 output
// channels, run as one conv_tc_kernel job per 128-channel N block and sub-pixel phase (csrc/net.cu, conv_plan.hpp:
// plan_conv_nblocks, conv_nblock_*).  Reuses the mirror of the slot chooser and the error state of conv_emu.cu.  Not part
// of libfav_b200.so.
#include "conv_emu.cu"

// A stylization-net convolution with Cout > 128 (net.cu): plan_conv_nblocks gives one ConvDef per N block -- the tap-paired
// first conv, generic stride-1, the parity-split stride-2 'd' conv, or the sub-pixel phases of a transposed 'u' / 'f' conv.
// Every (block, phase) job is planned, packed (conv_nblock_weights, transposed slices included) and addressed by the
// product's host code; the emulated kernel writes the raw output through the block's offset pointer and adds the fused
// InstanceNorm statistics through conv_nblock_stats into one [sum][sum of squares] array.  Checks: every raw element and
// every statistics slot is written by exactly one block, and both match a direct (transposed) convolution.
extern "C" int emu_style_nblock_check(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int H, int W,
                                      unsigned seed, double *max_err, double *max_ref, double *stats_err, int *n_jobs) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  std::vector<float> w((size_t)cout * cin * k * k), x((size_t)cin * H * W);
  for (auto &v : w) v = U(rng) * 0.05f;
  for (auto &v : x) v = U(rng) * 3.f;
  ConvDef c;  // as fav_net_create / fav_net_finalize build it
  init_conv_def(c, "l9", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  c.raw_out = true;
  if (plan_conv_nblocks(c) != FAV_OK) return 1;
  if ((int)c.nblock.size() != conv_nblocks(cout)) { set_error("%d N blocks planned", (int)c.nblock.size()); return 12; }
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
  const int Cq = round_up(cout, 4) / 4, Wp = round_up(Wo, kTileM);
  std::vector<double> raw((size_t)Ho * Cq * Wp * 4 + 4096, 0.0);  // + slack as build_plan allocates
  std::vector<int> written(raw.size(), 0);
  std::vector<double> sums(2 * cout + 2 * kMaxNBlock, 0.0);  // slack: a misplaced block must be caught, not crash
  std::vector<int> slot_block(sums.size(), -1);
  int jobs = 0;
  for (int b = 0; b < (int)c.nblock.size(); ++b) {
    const ConvDef &cb = c.nblock[b];
    const std::vector<float> wb = conv_nblock_weights(w, cin, cout, k, b, c.transposed);
    double *raw_b = raw.data() + conv_nblock_raw_offset(b, Wp);
    for (const ConvPhase &ph : cb.phases) {
      if (ph.kind == 3) { set_error("N-block job planned as x-fold"); return 12; }
      std::vector<uint16_t> pk = pack_phase_weights(cb, ph, wb);
      ConvJob j;
      if (fill_conv_job(cb, ph, op, j) != FAV_OK) return 2;
      j.raw_Cq = Cq; j.raw_Wp = Wp;  // build_conv_jobs: the whole tensor's pitches
      conv_nblock_stats(j, sums.data(), cout, b);
      conv_tc_choose_slots(j);
      if (conv_tc_smem_bytes(j) > 227 * 1024 || (!j.b_resident && j.b_slots < 2)) { set_error("smem budget"); return 3; }
      ++jobs;
      const int Npad = j.Npad;
      std::vector<uint16_t> st_hi((size_t)j.stage16 * 8), st_lo((size_t)j.stage16 * 8);
      std::vector<double> acc((size_t)kTileM * Npad);
      for (int tile = 0; tile < j.ntiles; ++tile) {
        const int y = tile / j.tiles_x, x0 = (tile % j.tiles_x) * j.tile_dx;
        std::fill(acc.begin(), acc.end(), 0.0);
        for (int g = 0; g < j.ngroups; ++g) {
          std::fill(st_hi.begin(), st_hi.end(), (uint16_t)0x7e00);  // NaN poison
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
          for (int ch = 0; ch < j.nchunks; ++ch) {
            const uint16_t *chunk = pk.data() + (size_t)(g * j.nchunks + ch) * j.chunk16 * 8;
            const uint16_t *b_hi = chunk, *b_lo = chunk + (size_t)j.spc * 2 * Npad * 8;
            for (int st = 0; st < j.spc; ++st) {
              const KStep ks = j.steps[ch * j.spc + st];
              for (int m = 0; m < kTileM; ++m)
                for (int u = 0; u < 2; ++u) {
                  int64_t a16 = (int64_t)ks.a_off16 + (int64_t)u * ks.lbo16 + m;
                  if (a16 >= j.stage16) { set_error("A desc OOB"); return 6; }
                  for (int i = 0; i < 8; ++i) {
                    double ah = h2f_bits(st_hi[a16 * 8 + i]), al = h2f_bits(st_lo[a16 * 8 + i]);
                    for (int n = 0; n < Npad; ++n) {
                      int64_t b16 = (int64_t)st * 2 * Npad + (int64_t)u * Npad + n;
                      double bh = h2f_bits(b_hi[b16 * 8 + i]), bl = h2f_bits(b_lo[b16 * 8 + i]);
                      acc[(size_t)m * Npad + n] += ah * bh + al * bh + ah * bl;
                    }
                  }
                }
            }
          }
        }
        // epilogue of conv_tc_kernel: raw store through the block's pointer, statistics through job.stats / stats_pitch
        for (int m = 0; m < kTileM; ++m) {
          const int xx = x0 + m;
          if (xx >= j.Wo || y >= j.Ho) continue;
          const int yo = y * j.oy_mul + j.oy_off, xo = xx * j.ox_mul + j.ox_off;
          for (int n = 0; n < j.Cout; ++n) {
            const int64_t o = (raw_b - raw.data()) + (((int64_t)yo * j.raw_Cq + (n >> 2)) * j.raw_Wp + xo) * 4 + (n & 3);
            if (o < 0 || o >= (int64_t)raw.size()) { set_error("raw OOB"); return 7; }
            const double v = acc[(size_t)m * Npad + n];
            raw[o] = v;
            written[o]++;
            for (int q = 0; q < 2; ++q) {
              const int64_t s = (j.stats - sums.data()) + (q ? j.stats_pitch : 0) + n;
              if (s < 0 || s >= (int64_t)sums.size()) { set_error("stats slot OOB"); return 9; }
              if (slot_block[s] >= 0 && slot_block[s] != b) { set_error("stats slot %lld shared by blocks %d and %d", (long long)s, slot_block[s], b); return 10; }
              slot_block[s] = b;
              sums[s] += q ? v * v : v;
            }
          }
        }
      }
    }
  }
  // direct reference
  std::vector<double> ref((size_t)cout * Ho * Wo, 0.0);
  if (!transposed) {
    for (int co = 0; co < cout; ++co)
      for (int oy = 0; oy < Ho; ++oy)
        for (int ox = 0; ox < Wo; ++ox) {
          double s = 0;
          for (int ci = 0; ci < cin; ++ci)
            for (int ky = 0; ky < k; ++ky) {
              const int iy = oy * stride + ky - pad;
              if (iy < 0 || iy >= H) continue;
              for (int kx = 0; kx < k; ++kx) {
                const int ix = ox * stride + kx - pad;
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
          const double xv = xq[((size_t)ci * H + iy) * W + ix];
          for (int ky = 0; ky < k; ++ky) {
            const int oy = iy * stride - pad + ky;
            if (oy < 0 || oy >= Ho) continue;
            for (int kx = 0; kx < k; ++kx) {
              const int ox = ix * stride - pad + kx;
              if (ox < 0 || ox >= Wo) continue;
              for (int co = 0; co < cout; ++co)
                ref[((size_t)co * Ho + oy) * Wo + ox] += xv * w[(((size_t)ci * cout + co) * k + ky) * k + kx];
            }
          }
        }
  }
  double me = 0, mr = 0, se = 0;
  for (int co = 0; co < cout; ++co) {
    double s1 = 0, s2 = 0, a1 = 0, a2 = 0;
    for (int oy = 0; oy < Ho; ++oy)
      for (int ox = 0; ox < Wo; ++ox) {
        const double r = ref[((size_t)co * Ho + oy) * Wo + ox];
        const size_t o = (((size_t)oy * Cq + co / 4) * Wp + ox) * 4 + co % 4;
        if (written[o] != 1) { set_error("raw element (c %d, y %d, x %d) written %d times", co, oy, ox, written[o]); return 8; }
        double d = std::fabs(raw[o] - r);
        if (!(d <= 1e300)) d = 1e300;
        me = std::max(me, d);
        mr = std::max(mr, std::fabs(r));
        s1 += r; s2 += r * r; a1 += std::fabs(r); a2 += r * r;
      }
    if (slot_block[co] < 0 || slot_block[cout + co] < 0) { set_error("statistics of channel %d never written", co); return 11; }
    double d1 = std::fabs(sums[co] - s1) / std::max(a1, 1.0), d2 = std::fabs(sums[cout + co] - s2) / std::max(a2, 1.0);
    if (!(d1 <= 1e300)) d1 = 1e300;
    if (!(d2 <= 1e300)) d2 = 1e300;
    se = std::max(se, std::max(d1, d2));
  }
  for (size_t s = 2 * (size_t)cout; s < sums.size(); ++s)
    if (slot_block[s] >= 0) { set_error("statistics slot %zu beyond the tensor's 2 x %d written", s, cout); return 11; }
  *max_err = me; *max_ref = mr; *stats_err = se;
  if (n_jobs) *n_jobs = jobs;
  return 0;
}
