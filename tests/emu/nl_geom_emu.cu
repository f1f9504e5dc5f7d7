// nl_geom_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of the norm-on-load patch producers of conv_tc_kernel (warps 9-12),
// checked against the patch the bulk copies stage from the operand in_apply writes.  The jobs come from the product's planner
// (plan_conv_nblocks, operand_geometry, fill_conv_job, set_conv_batch, set_norm_on_load, nl_geometry_ok in conv_plan.hpp and
// conv.cuh), the producer's addressing from the helpers the kernel calls (tile_at, nl_raw_row, nl_raw_col).  Not part of
// libfav_b200.so.
#include "conv_emu.cu"

namespace {
struct Raw {  // a raw conv output [B][H][Cq][Wp][4], with non-zero junk in the columns x >= W the kernel never reads
  RawTensor t;
  std::vector<float> v;
};
// the same value function on both sides: InstanceNorm (+ReLU) of channel c of image b, then the fp16 hi / lo split
struct Norm {
  std::vector<float> mean, scale, beta;  // [B][C]
  int C = 0, relu = 1;
  void apply(const float *x, int b, int cb, uint16_t hi[8], uint16_t lo[8]) const {
    for (int i = 0; i < 8; ++i) {
      const int c = b * C + cb * 8 + i;
      float t = (x[i] - mean[c]) * scale[c] + beta[c];
      if (relu) t = std::max(t, 0.f);
      hi[i] = f2h_bits(t);
      lo[i] = f2h_bits(t - h2f_bits(hi[i]));
    }
  }
};
int fail(int code, const char *fmt, int layer, int a, int b, int c) {
  char buf[256];
  snprintf(buf, sizeof(buf), fmt, layer, a, b, c);
  set_error("%s", buf);
  return code;
}
}  // namespace

// rows: n x 8 ints as emu_batch_check reads them (batch_emu.cu): {type, cin, cout, k, stride, pad, transposed, adj}, type 0 =
// conv, 1 = nearest upsampling by `stride`, 2 = first conv of an R/C block, 3 = second conv of an R block, 4 = second conv of a
// C block; the last row is the final convolution.  in_H / in_W: the net input including the reflection padding.  B images.
// A convolution normalises on load as build_plan decides (net.cu fuse_norm_on_load): its input is a plain InstanceNorm output
// (the previous row is a conv whose norm adds no skip), no later step reads that operand as a skip (not the first conv of an R
// block), at most 256 channels, and every job has a patch layout nl_geometry_ok accepts.  For each such job, every (image,
// tile, group, patch row, channel block, pixel) of the stage the producers fill is compared, hi and lo, byte for byte with the
// stage the bulk copies fill from the in_apply'd operand.  The only pixels allowed to differ are those whose bulk source lies
// past the end of its (row, channel block) slab -- the next slab's data, which the bulk copy stages and the producer zeroes:
// they must lie outside the image and beyond every pixel a stored output reads.
// info[4]: fused convolutions, fused jobs, compared pixels (16-byte cells of hi and of lo), pixels past a slab end.
extern "C" int emu_nl_geometry_check(int n, const int *rows, int in_H, int in_W, int B, unsigned seed, int *info) {
  std::vector<ConvDef> convs(n);
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) continue;
    init_conv_def(convs[r], "l" + std::to_string(r), d[1], d[2], d[3], d[4], d[5], d[6] != 0, d[7]);
    build_phases(convs[r]);
    convs[r].raw_out = r + 1 < n;
    if (plan_conv_nblocks(convs[r]) != FAV_OK) return 1;
  }
  auto next_conv = [&](int r) -> const ConvDef * {
    for (int q = r + 1; q < n; ++q)
      if (rows[8 * q] != 1) return &convs[q];
    return nullptr;
  };
  for (int i = 0; i < 4; ++i) info[i] = 0;
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-3.f, 3.f);
  Operand cur = operand_geometry(rows[1], in_H, in_W, next_conv(-1));
  Raw prev;               // raw output of the previous row's conv (empty after an upsampling)
  bool prev_plain = false;  // its norm adds no skip
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) {
      cur = operand_geometry(cur.C, cur.H * d[4], cur.W * d[4], next_conv(r));
      prev_plain = false;
      continue;
    }
    const ConvDef &c = convs[r];
    const bool last = r + 1 == n;
    int ho, wo;
    conv_out_size(c, cur.H, cur.W, &ho, &wo);
    cur.img16 = (int64_t)cur.elems16;
    const bool src_is_skip = d[0] == 2 && r + 1 < n && rows[8 * (r + 1)] == 3;
    std::vector<ConvJob> jobs;
    bool fuse = prev_plain && !src_is_skip && c.cin <= 256;
    const int nb = c.nblock.empty() ? 1 : (int)c.nblock.size();
    for (int blk = 0; blk < nb && fuse; ++blk) {
      const ConvDef &cd = c.nblock.empty() ? c : c.nblock[blk];
      for (const ConvPhase &ph : cd.phases) {
        ConvJob j;
        if (fill_conv_job(cd, ph, cur, j) != FAV_OK) return 2;
        set_conv_batch(j, B, 0, 0, 0);
        set_norm_on_load(j, prev.t, cur, 1, nullptr, 2 * c.cin, nullptr, nullptr);
        if (!nl_geometry_ok(j)) { fuse = false; break; }
        jobs.push_back(j);
      }
    }
    if (fuse) {
      ++info[0];
      // the producer's statistics table and the operand in_apply writes from prev (zero border, interior pixels only)
      Norm nm;
      nm.C = c.cin;
      for (int i = 0; i < B * c.cin; ++i) {
        nm.mean.push_back(U(rng) * 0.3f);
        nm.scale.push_back(0.2f + std::fabs(U(rng)));
        nm.beta.push_back(U(rng) * 0.5f);
      }
      const int64_t cells = (int64_t)B * cur.img16;
      std::vector<uint16_t> ohi((size_t)cells * 8, 0), olo((size_t)cells * 8, 0);
      for (int b = 0; b < B; ++b)
        for (int y = 0; y < prev.t.H; ++y)
          for (int cb = 0; cb < cur.Cb; ++cb)
            for (int x = 0; x < prev.t.W; ++x) {
              float v[8];
              for (int i = 0; i < 8; ++i) v[i] = prev.v[b * prev.t.img + prev.t.off4(y, 2 * cb + i / 4, x) * 4 + i % 4];
              const int64_t o = (b * cur.img16 + cur.off16(cur.padT + y, cb, cur.padL + x)) * 8;
              nm.apply(v, b, cb, &ohi[o], &olo[o]);
            }
      for (const ConvJob &j : jobs) {
        ++info[1];
        const int total = B * j.ntiles;
        for (int T = 0; T < total; ++T) {
          const TileAt at = tile_at(j, T);
          const int nvalid = std::min(j.tile_dx, j.Wo - at.x0);
          for (int g = 0; g < j.ngroups; ++g)
            for (int ri = 0; ri < j.nrows; ++ri)
              for (int cbi = 0; cbi < j.CbG; ++cbi) {
                const int cb = j.grp_cb0[g] + cbi, ry = nl_raw_row(j, at.y, g, ri);
                const int64_t srow = ((int64_t)(j.row_mul * at.y + j.grp_row[g][ri]) * j.a_Cb + cb) * j.a_slab16;
                for (int p = 0; p < j.pslab16; ++p) {
                  // the bulk copies: segment `seg` covers stage pixels [seg_dst16, seg_dst16 + seg_len16)
                  const int seg = j.nseg == 2 && p >= j.seg_dst16[1] ? 1 : 0;
                  const int scol = j.seg_src16[seg] + at.x0 + (p - j.seg_dst16[seg]);
                  const int64_t s16 = srow + scol + at.a16;
                  if (s16 < 0 || s16 >= cells) return fail(3, "layer %d: bulk source outside the operand (tile %d, group %d, pixel %d)", r, T, g, p);
                  // the producer
                  uint16_t hi[8] = {0}, lo[8] = {0};
                  const int x = nl_raw_col(j, at.x0, p);
                  if (ry >= 0 && ry < j.nl_H && x >= 0 && x < j.nl_W) {
                    float v[8];
                    for (int i = 0; i < 8; ++i)
                      v[i] = prev.v[at.nl_raw4 * 4 + (((int64_t)ry * j.nl_Cq + 2 * cb + i / 4) * j.nl_Wp + x) * 4 + i % 4];
                    nm.apply(v, at.b, cb, hi, lo);
                  }
                  ++info[2];
                  if (!memcmp(hi, &ohi[s16 * 8], 16) && !memcmp(lo, &olo[s16 * 8], 16)) continue;
                  // a pixel past the end of its slab: outside the image, zero, and read by no stored output
                  const int reach = j.nseg == 2 ? (seg ? j.seg_dst16[1] + nvalid - 1 : nvalid)
                                                : nvalid - 1 + (j.xfold_kw ? j.xfold_kw - 1 : j.pslab16 - kTileM);
                  bool zero = true;
                  for (int i = 0; i < 8; ++i) zero = zero && !hi[i] && !lo[i];
                  if (scol >= j.a_slab16 && zero && (x < 0 || x >= j.nl_W) && p > reach) { ++info[3]; continue; }
                  char what[96];
                  snprintf(what, sizeof(what), "layer %%d: stage differs (tile %%d, group %%d, pixel %%d; row %d, cb %d, raw x %d)", ri, cb, x);
                  return fail(4, what, r, T, g, p);
                }
              }
        }
      }
    }
    if (last) break;
    // this conv's raw output, read by the next row when it normalises on load
    prev.t = RawTensor();
    prev.t.C = c.cout; prev.t.Cq = round_up(c.cout, 4) / 4; prev.t.H = ho; prev.t.W = wo; prev.t.Hp = ho + 2;
    prev.t.Wp = round_up(wo, kTileM);
    prev.t.img = (int64_t)prev.t.Hp * prev.t.Cq * prev.t.Wp * 4 + 1024;
    prev.v.assign((size_t)(B * prev.t.img), 0.f);
    for (float &v : prev.v) v = U(rng);
    prev_plain = d[0] != 3;
    cur = operand_geometry(c.cout, ho, wo, next_conv(r));
  }
  return 0;
}
