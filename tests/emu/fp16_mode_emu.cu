// fp16_mode_emu.cu -- TEST INFRASTRUCTURE: a CPU emulation of conv_tc_kernel's single pass (ConvJob::single, PAIR == false),
// on the jobs the product's planner builds (conv_plan.hpp).  The patch producer's bulk copies (its copy loop with one plane)
// and the weight producer's copy of each chunk's first half land in stages and slots poisoned with NaNs; the consumer reads
// them through the kernel's descriptor addressing (hi planes only).  Checked: the bytes each producer announces (tc_a_stage_tx,
// FAV_TC_B_CHUNK_TX, conv.cuh) equal the bytes it copies, and the hi prefix of every packed chunk holds exactly the hi steps
// the consumer reads: the result equals, to fp64 rounding, a direct convolution of fp16(x) with the fp16 hi weights.
// Also exports those hi weights (weight_half, set_weight_prescale) for the oracle's emulation of the mode.
// Not part of libfav_b200.so.
#include "conv_emu.cu"

// hi weights of a convolution as the product packs them, back in weight units: fp16(w 2^e) 2^-e, e = ConvDef::w_exp
extern "C" int emu_fp16_weight_hi(int cin, int cout, int k, int stride, int pad, int transposed, int adj, const float *w,
                                  double *out, int *e_out) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  const size_t n = (size_t)cin * cout * k * k;
  std::vector<float> wv(w, w + n);
  set_weight_prescale(c, wv);
  for (size_t i = 0; i < n; ++i) out[i] = std::ldexp((double)h2f_bits(weight_half(wv[i], c.w_exp, 0)), -c.w_exp);
  *e_out = c.w_exp;
  return 0;
}

// mode 0: one job per sub-pixel phase (or the plain conv), split into N blocks when Cout > 128; 1: the stacked-phase jobs
// (plan_phase_stack).  nimg: images of one launch (tile_at).  out: [0] max |emulated - direct| / max(1, max |direct|),
// [1] jobs, [2] A bytes announced per stage summed over jobs, [3] B bytes announced per chunk summed over jobs, [4] the norm-on-load
// geometry (nl_geometry_ok) of the first job
extern "C" int emu_fp16_conv_check(int cin, int cout, int k, int stride, int pad, int transposed, int adj, int H, int W, int mode,
                                   int nimg, unsigned seed, double *out) {
  ConvDef c;
  init_conv_def(c, "emu", cin, cout, k, stride, pad, transposed != 0, adj);
  build_phases(c);
  if (plan_conv_nblocks(c) != FAV_OK) return 1;
  if (mode == 1 && (plan_phase_stack(c) != FAV_OK || c.stack.empty())) { set_error("no stacked-phase plan"); return 1; }
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  std::vector<float> w((size_t)cin * cout * k * k), x((size_t)nimg * cin * H * W);
  for (auto &v : w) v = U(rng) * 0.1f;
  for (auto &v : x) v = U(rng) * 3.f;
  Operand op = operand_geometry(cin, H, W, &c);
  const int64_t img16 = (int64_t)op.elems16;
  std::vector<uint16_t> hi((size_t)nimg * img16 * 8, 0);
  std::vector<double> xq(x.size());
  for (int b = 0; b < nimg; ++b)
    for (int ci = 0; ci < cin; ++ci)
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          const size_t i = (((size_t)b * cin + ci) * H + y) * W + xx;
          const uint16_t hb = f2h_bits(x[i]);
          hi[(size_t)(b * img16 + op.off16(op.padT + y, ci / 8, op.padL + xx)) * 8 + ci % 8] = hb;
          xq[i] = h2f_bits(hb);
        }
  int Ho, Wo;
  conv_out_size(c, H, W, &Ho, &Wo);
  std::vector<double> got((size_t)nimg * cout * Ho * Wo, std::nan("")), ref(got.size(), 0.0);
  set_weight_prescale(c, w);
  std::vector<double> whi(w.size());
  for (size_t i = 0; i < w.size(); ++i) whi[i] = std::ldexp((double)h2f_bits(weight_half(w[i], c.w_exp, 0)), -c.w_exp);
  // the jobs: (ConvDef, phase, weights, first output channel, accumulator column -> (phase, channel))
  struct J { const ConvDef *cd; const ConvPhase *ph; std::vector<float> w; int co0; };
  std::vector<J> jobs;
  if (mode == 1) {
    for (const ConvPhase &ph : c.stack) jobs.push_back(J{&c, &ph, w, 0});
  } else if (!c.nblock.empty()) {
    for (int b = 0; b < (int)c.nblock.size(); ++b)
      for (const ConvPhase &ph : c.nblock[b].phases)
        jobs.push_back(J{&c.nblock[b], &ph, conv_nblock_weights(w, cin, cout, k, b, c.transposed), b * kMaxNBlock});
  } else {
    for (const ConvPhase &ph : c.phases) jobs.push_back(J{&c, &ph, w, 0});
  }
  double a_tx_sum = 0, b_tx_sum = 0;
  int nl_ok = -1;
  for (J &jb : jobs) {
    ConvDef cd = *jb.cd;
    cd.w_exp = c.w_exp;  // every job of a conv runs with the conv's exponent
    const std::vector<uint16_t> pk = pack_phase_weights(cd, *jb.ph, jb.w);
    ConvJob j;
    if (fill_conv_job(cd, *jb.ph, op, j) != FAV_OK) return 2;
    j.single = 1;
    j.nimg = nimg; j.a_img16 = img16;
    conv_tc_choose_slots(j);
    if (nl_ok < 0) nl_ok = nl_geometry_ok(j) ? 1 : 0;
    const int Npad = j.Npad, NT = Npad;
    const uint32_t a_tx = tc_a_stage_tx(j, false), chunk_bytes = (uint32_t)j.chunk16 * 16u;
    const uint32_t b_tx = FAV_TC_B_CHUNK_TX(j.dbg, chunk_bytes, false);
    a_tx_sum += a_tx; b_tx_sum += b_tx;
    if ((size_t)j.ngroups * j.nchunks * j.chunk16 * 8 != pk.size()) { set_error("packed size %zu != jobs' chunks", pk.size()); return 3; }
    // one stage: hi plane then lo plane (a_stage_bytes each); one slot: chunk_bytes
    std::vector<uint16_t> stage((size_t)2 * j.stage16 * 8), slot((size_t)j.chunk16 * 8);
    std::vector<double> acc((size_t)kTileM * Npad);
    for (int T = 0; T < nimg * j.ntiles; ++T) {
      const TileAt at = tile_at(j, T, true);
      std::fill(acc.begin(), acc.end(), 0.0);
      for (int g = 0; g < j.ngroups; ++g) {
        // A producer (conv_tc.cu, warp kAWarp, NP = 1)
        std::fill(stage.begin(), stage.end(), (uint16_t)0x7e00);
        const int NP = 1, per_row = j.CbG * j.nseg * NP, ncopies = j.nrows * per_row;
        uint64_t copied = 0;
        for (int cp = 0; cp < ncopies; ++cp) {
          int ri = cp / per_row, r = cp - ri * per_row;
          int cbi = r / (j.nseg * NP);
          r -= cbi * j.nseg * NP;
          const int seg = r, part = 0;
          const int64_t src16 = ((int64_t)(j.row_mul * at.y + j.grp_row[g][ri]) * j.a_Cb + j.grp_cb0[g] + cbi) * j.a_slab16 +
                                j.seg_src16[seg] + at.x0 + at.a16;
          const int64_t dst16 = (int64_t)part * j.stage16 + (int64_t)(ri * j.CbG + cbi) * j.pslab16 + j.seg_dst16[seg];
          const int len = j.seg_len16[seg];
          if (src16 < 0 || src16 + len > (int64_t)nimg * img16) { set_error("patch copy outside the operand"); return 4; }
          if (dst16 + len > j.stage16) { set_error("patch copy outside the hi plane of the stage"); return 5; }
          std::copy(hi.begin() + src16 * 8, hi.begin() + (src16 + len) * 8, stage.begin() + dst16 * 8);
          copied += (uint64_t)len * 16;
        }
        if (copied != a_tx) { set_error("A producer copies %llu bytes, announces %u", (unsigned long long)copied, a_tx); return 6; }
        for (int ch = 0; ch < j.nchunks; ++ch) {
          // B producer: the first b_tx bytes of the chunk
          std::fill(slot.begin(), slot.end(), (uint16_t)0x7e00);
          const uint16_t *src = pk.data() + (size_t)(g * j.nchunks + ch) * j.chunk16 * 8;
          std::copy(src, src + b_tx / 2, slot.begin());
          // consumer: per K step, the hi descriptors only (a_hi16 + a_off16, bs = slot + st * b_step16)
          const uint32_t b_step16 = 2u * (uint32_t)NT;
          for (int st = 0; st < j.spc; ++st) {
            const KStep ks = j.steps[ch * j.spc + st];
            for (int m = 0; m < kTileM; ++m)
              for (int u = 0; u < 2; ++u) {
                const int64_t a16 = (int64_t)ks.a_off16 + (int64_t)u * ks.lbo16 + m;
                if (a16 >= j.stage16) { set_error("A descriptor outside the hi plane"); return 7; }
                for (int i = 0; i < 8; ++i) {
                  const double a = h2f_bits(stage[a16 * 8 + i]);
                  for (int n = 0; n < Npad; ++n) {
                    const int64_t b16 = (int64_t)st * b_step16 + (int64_t)u * NT + n;
                    if ((b16 + 1) * 16 > (int64_t)b_tx) { set_error("B descriptor past the copied hi prefix"); return 8; }
                    acc[(size_t)m * Npad + n] += a * h2f_bits(slot[b16 * 8 + i]);
                  }
                }
              }
          }
        }
      }
      // placement (the kernel's epilogues, without the bias): plain / x-fold / stacked phases
      for (int m = 0; m < kTileM; ++m) {
        const int xx = at.x0 + m;
        if (xx >= j.Wo || at.y >= j.Ho) continue;
        if (j.xfold_kw) {
          if (m >= j.tile_dx) continue;
          for (int n = 0; n < j.Cout; ++n) {
            double s = 0;
            for (int kx = 0; kx < j.xfold_kw; ++kx) s += acc[(size_t)(m + kx) * Npad + kx * j.Cout + n];
            got[(((size_t)at.b * cout + n) * Ho + at.y) * Wo + xx] = s * j.w_unscale;
          }
          continue;
        }
        const int ns = j.nstack ? j.nstack : 1;
        for (int s = 0; s < ns; ++s) {
          const int yo = at.y * j.oy_mul + (j.nstack ? j.st_oy[s] : j.oy_off);
          const int xo = xx * j.ox_mul + (j.nstack ? j.st_ox[s] : j.ox_off);
          if (yo >= Ho || xo >= Wo) { set_error("output outside the grid"); return 9; }
          for (int n = 0; n < j.Cout; ++n)
            got[(((size_t)at.b * cout + jb.co0 + n) * Ho + yo) * Wo + xo] = acc[(size_t)m * Npad + s * j.Cout + n] * j.w_unscale;
        }
      }
    }
  }
  // direct convolution of fp16(x) with the hi weights, fp64
  for (int b = 0; b < nimg; ++b)
    for (int ci = 0; ci < cin; ++ci)
      for (int iy = 0; iy < H; ++iy)
        for (int ix = 0; ix < W; ++ix) {
          const double xv = xq[(((size_t)b * cin + ci) * H + iy) * W + ix];
          for (int ky = 0; ky < k; ++ky)
            for (int kx = 0; kx < k; ++kx)
              for (int co = 0; co < cout; ++co) {
                int oy, ox;
                double wv;
                if (!transposed) {  // out(oy, ox) += w x(oy * s + ky - pad, ...): scatter form
                  if ((iy + pad - ky) % stride || (ix + pad - kx) % stride) continue;
                  oy = (iy + pad - ky) / stride; ox = (ix + pad - kx) / stride;
                  if (iy + pad - ky < 0 || ix + pad - kx < 0) continue;
                  wv = whi[(((size_t)co * cin + ci) * k + ky) * k + kx];
                } else {
                  oy = iy * stride - pad + ky; ox = ix * stride - pad + kx;
                  wv = whi[(((size_t)ci * cout + co) * k + ky) * k + kx];
                }
                if (oy < 0 || oy >= Ho || ox < 0 || ox >= Wo) continue;
                ref[(((size_t)b * cout + co) * Ho + oy) * Wo + ox] += xv * wv;
              }
        }
  double me = 0, mr = 0;
  for (size_t i = 0; i < ref.size(); ++i) {
    double d = std::fabs(got[i] - ref[i]);
    if (!(d <= 1e300)) d = 1e300;
    me = std::max(me, d);
    mr = std::max(mr, std::fabs(ref[i]));
  }
  out[0] = me / std::max(1.0, mr); out[1] = (double)jobs.size(); out[2] = a_tx_sum; out[3] = b_tx_sum; out[4] = nl_ok;
  return 0;
}
