// nblock_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of a convolution with more than 128 output channels run as one
// conv_tc_kernel job per 128-channel N block (conv_plan.hpp: conv_nblock_*), as the loss network of -evaluate does
// (csrc/percep.cu).  Each block is planned, packed and addressed by the product's own host code; the emulated kernel
// writes the raw [Ho][Cq][Wp][4] output through the block's offset pointer, and the whole tensor is compared against a
// direct convolution.  Reuses the mirror of the slot chooser and the error state of conv_emu.cu.  Not part of libfav_b200.so.
#include "conv_emu.cu"

extern "C" int emu_nblock_check(int cin, int cout, int k, int pad, int H, int W, unsigned seed, double *max_err, double *max_ref,
                                int *n_jobs, int *max_groups) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  std::vector<float> w((size_t)cout * cin * k * k), x((size_t)cin * H * W);
  for (auto &v : w) v = U(rng) * 0.05f;
  for (auto &v : x) v = U(rng) * 3.f;
  const int nb = conv_nblocks(cout);
  ConvDef c0;
  init_conv_def(c0, "emu", cin, conv_nblock_cout(cout, 0), k, 1, pad, false, 0);
  build_phases(c0);
  Operand op = operand_geometry(cin, H, W, &c0);
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
  conv_out_size(c0, H, W, &Ho, &Wo);
  const int Cq = round_up(cout, 4) / 4, Wp = round_up(Wo, kTileM);
  std::vector<double> raw((size_t)Ho * Cq * Wp * 4, 0.0);
  std::vector<int> written(raw.size(), 0);
  int groups = 0;
  for (int b = 0; b < nb; ++b) {
    ConvDef c;
    init_conv_def(c, "emu", cin, conv_nblock_cout(cout, b), k, 1, pad, false, 0);
    build_phases(c);
    ConvPhase &ph = c.phases[0];
    if (build_phase_tables(c, ph) != FAV_OK) return 1;
    if (ph.kind != 0 && ph.kind != 1) { set_error("N-block job planned as kind %d", ph.kind); return 12; }
    const std::vector<float> wb = conv_nblock_weights(w, cin, cout, k, b);
    std::vector<uint16_t> pk = pack_phase_weights(c, ph, wb);
    ConvJob j;
    if (fill_conv_job(c, ph, op, j) != FAV_OK) return 2;
    conv_tc_choose_slots(j);
    if (conv_tc_smem_bytes(j) > 227 * 1024 || (!j.b_resident && j.b_slots < 2)) { set_error("smem budget"); return 3; }
    groups = std::max(groups, j.ngroups);
    const int Npad = j.Npad;
    const int64_t raw_off = conv_nblock_raw_offset(b, Wp);
    std::vector<uint16_t> st_hi((size_t)j.stage16 * 8), st_lo((size_t)j.stage16 * 8);
    std::vector<double> acc((size_t)kTileM * Npad);
    for (int tile = 0; tile < j.ntiles; ++tile) {
      const int y = tile / j.tiles_x, x0 = (tile % j.tiles_x) * j.tile_dx;
      std::fill(acc.begin(), acc.end(), 0.0);
      for (int g = 0; g < j.ngroups; ++g) {
        std::fill(st_hi.begin(), st_hi.end(), (uint16_t)0x7e00);  // NaN poison
        std::fill(st_lo.begin(), st_lo.end(), (uint16_t)0x7e00);
        for (int ri = 0; ri < j.nrows; ++ri)
          for (int cbi = 0; cbi < j.CbG; ++cbi) {
            int64_t src16 = ((int64_t)(j.row_mul * y + j.grp_row[g][ri]) * j.a_Cb + j.grp_cb0[g] + cbi) * j.a_slab16 + j.seg_src16[0] + x0;
            int64_t dst16 = (int64_t)(ri * j.CbG + cbi) * j.pslab16 + j.seg_dst16[0];
            if (src16 < 0 || src16 + j.seg_len16[0] > (int64_t)op.elems16) { set_error("src OOB"); return 4; }
            if (dst16 + j.seg_len16[0] > j.stage16) { set_error("dst OOB"); return 5; }
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
      // epilogue of conv_tc_kernel: channel c of the block -> raw + raw_off at ((yo * raw_Cq + c / 4) * raw_Wp + xo) * 4 + c % 4
      for (int m = 0; m < kTileM; ++m) {
        const int xx = x0 + m;
        if (xx >= j.Wo || y >= j.Ho) continue;
        for (int n = 0; n < j.Cout; ++n) {
          const int64_t o = raw_off + (((int64_t)y * Cq + (n >> 2)) * Wp + xx) * 4 + (n & 3);
          if (o < 0 || o >= (int64_t)raw.size()) { set_error("raw OOB"); return 7; }
          raw[o] = acc[(size_t)m * Npad + n];
          written[o]++;
        }
      }
    }
  }
  double me = 0, mr = 0;
  for (int co = 0; co < cout; ++co)
    for (int oy = 0; oy < Ho; ++oy)
      for (int ox = 0; ox < Wo; ++ox) {
        double s = 0;
        for (int ci = 0; ci < cin; ++ci)
          for (int ky = 0; ky < k; ++ky) {
            const int iy = oy + ky - pad;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < k; ++kx) {
              const int ix = ox + kx - pad;
              if (ix < 0 || ix >= W) continue;
              s += (double)w[(((size_t)co * cin + ci) * k + ky) * k + kx] * xq[((size_t)ci * H + iy) * W + ix];
            }
          }
        const size_t o = (((size_t)oy * Cq + co / 4) * Wp + ox) * 4 + co % 4;
        if (written[o] != 1) { set_error("raw element (c %d, y %d, x %d) written %d times", co, oy, ox, written[o]); return 8; }
        double d = std::fabs(raw[o] - s);
        if (!(d <= 1e300)) d = 1e300;
        me = std::max(me, d);
        mr = std::max(mr, std::fabs(s));
      }
  *max_err = me; *max_ref = mr;
  if (n_jobs) *n_jobs = nb;
  if (max_groups) *max_groups = groups;
  return 0;
}
