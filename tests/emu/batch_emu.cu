// batch_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of how conv_tc_kernel walks a BATCH of images (ConvJob::nimg) over every
// convolution of a net's plan.  The jobs come from the product's planner (plan_conv_nblocks, operand_geometry, fill_conv_job,
// set_conv_batch, set_opnd_epilogue in conv_plan.hpp), the tile decode and per-image base offsets from the helper every role of
// the kernel calls (tile_at, conv.cuh) and the operand-epilogue stores from opnd_epi_addr.  Not part of libfav_b200.so.
#include <set>

#include "conv_emu.cu"

namespace {
struct Span {  // one image's region of a tensor: [b * img, b * img + img)
  int64_t img;
  bool inside(int b, int64_t lo, int64_t hi_excl) const { return lo >= (int64_t)b * img && hi_excl <= (int64_t)(b + 1) * img; }
};
int fail(int code, const char *fmt, int layer, int b, int t) {
  char buf[256];
  snprintf(buf, sizeof(buf), fmt, layer, b, t);
  set_error("%s", buf);
  return code;
}
}  // namespace

// rows: n x 8 ints as emu_opnd_epi_check reads them (opnd_epi_emu.cu): {type, cin, cout, k, stride, pad, transposed, adj}, type
// 0 = conv, 1 = nearest upsampling by `stride`, 2 = first conv of an R/C block, 3 = second conv of an R block, 4 = second conv of
// a C block; the last row is the final convolution.  bn: batch-normalized net (operand epilogues, no raw tensors / statistics);
// else InstanceNorm with fused statistics and norm-on-load on the second conv of each block, as net.cu plans them.  in_H / in_W:
// the net input including the reflection padding; out_H / out_W: the frame.  For every tensor-core job of a batch of B images on
// num_sms persistent CTAs, checked:
//   1. every (image, tile) is run by exactly one CTA;
//   2. each CTA's ordered tiles of image b are the ordered tiles some CTA runs when that image runs alone (nimg = 1);
//   3. every address of image b -- patch reads of the A operand or of the raw tensor it normalises on load, raw and statistics
//      writes, operand-epilogue stores and skip reads, the final frame -- lies inside image b's region of its tensor.
// info[4]: jobs, jobs normalising on load, jobs with an operand epilogue, jobs whose batch grid spans more CTAs than one image's.
extern "C" int emu_batch_check(int n, const int *rows, int in_H, int in_W, int out_H, int out_W, int bn, int B, int num_sms,
                               int *info) {
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
  // pass 1 as build_plan: per-image raw size (the largest raw tensor) and statistics slots
  int64_t raw_max = 0, stats_slots = 0;
  {
    int h = in_H, w = in_W;
    for (int r = 0; r < n; ++r) {
      const int *d = rows + 8 * r;
      if (d[0] == 1) { h *= d[4]; w *= d[4]; stats_slots += bn ? 0 : 2 * d[1]; continue; }
      int ho, wo;
      conv_out_size(convs[r], h, w, &ho, &wo);
      raw_max = std::max<int64_t>(raw_max, (int64_t)(ho + 2) * round_up(convs[r].cout, 4) * round_up(wo, kTileM));
      h = ho; w = wo;
      if (r + 1 < n && !bn) stats_slots += 2 * convs[r].cout;
    }
  }
  const int64_t raw_img = raw_max + 1024, stats_img = std::max<int64_t>(1, stats_slots), out_img = 3ll * out_H * out_W;
  std::vector<Operand> ops;
  ops.push_back(operand_geometry(rows[1], in_H, in_W, next_conv(-1)));
  int cur = 0, block_in = -1, stats_off = 0;
  RawTensor prev_raw;
  int prev_stats = -1;
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) {
      ops.push_back(operand_geometry(ops[cur].C, ops[cur].H * d[4], ops[cur].W * d[4], next_conv(r)));
      cur = (int)ops.size() - 1;
      if (!bn) stats_off += 2 * d[1];
      continue;
    }
    const ConvDef &c = convs[r];
    const bool last = r + 1 == n;
    if (d[0] == 2) block_in = cur;
    int ho, wo;
    conv_out_size(c, ops[cur].H, ops[cur].W, &ho, &wo);
    for (Operand &o : ops) o.img16 = (int64_t)o.elems16;
    RawTensor raw;
    raw.C = c.cout; raw.Cq = round_up(c.cout, 4) / 4; raw.H = ho; raw.W = wo; raw.Hp = ho + 2; raw.Wp = round_up(wo, kTileM);
    raw.img = raw_img;
    Operand dst;
    if (!last) { dst = operand_geometry(c.cout, ho, wo, next_conv(r)); dst.img16 = (int64_t)dst.elems16; }
    const Operand src = ops[cur];
    const bool skip = d[0] == 3;
    const int shave = c.pad == 0 ? 2 : 0;
    // norm-on-load (net.cu): the second conv of a block, when the first conv's norm has no skip and at most 256 channels
    const bool try_nl = !bn && (d[0] == 3 || d[0] == 4) && c.cin <= 256;
    const int nb = c.nblock.empty() ? 1 : (int)c.nblock.size();
    for (int blk = 0; blk < nb; ++blk) {
      const ConvDef &cd = c.nblock.empty() ? c : c.nblock[blk];
      std::vector<const ConvPhase *> phs;
      if (cd.has_fold) phs.push_back(&cd.fold);
      else for (const ConvPhase &ph : cd.phases) phs.push_back(&ph);
      for (const ConvPhase *ph : phs) {
        ConvJob j;
        if (fill_conv_job(cd, *ph, src, j) != FAV_OK) return 2;
        set_conv_batch(j, B, raw.img, out_img, stats_img);
        if (!last) j.final_mode = 0; else j.final_mode = 1;
        const int64_t raw0 = conv_nblock_raw_offset(blk, raw.Wp);
        j.raw_Cq = raw.Cq; j.raw_Wp = raw.Wp;
        const int64_t st0 = stats_off + (int64_t)blk * kMaxNBlock;
        if (!last && bn) set_opnd_epilogue(j, blk, nullptr, dst, d[0] != 3, skip ? &ops[block_in] : nullptr, shave);
        if (try_nl && !j.rf_R && !j.pf && !j.xfold_kw && j.nseg == 1 && j.seg_dst16[0] == 0 && j.seg_len16[0] == j.pslab16 &&
            j.row_mul == 1) {
          j.nl = 1; j.nl_Cq = prev_raw.Cq; j.nl_Wp = prev_raw.Wp; j.nl_H = prev_raw.H; j.nl_W = prev_raw.W;
          j.nl_padT = src.padT; j.nl_padL = src.padL; j.nl_C = c.cin;
          j.nl_raw_img4 = prev_raw.img / 4; j.nl_sums_img = stats_img;
        }
        ++info[0];
        info[1] += j.nl;
        info[2] += j.opnd;
        const int total = B * j.ntiles, G = std::min(total, num_sms), G1 = std::min(j.ntiles, num_sms);
        info[3] += G > G1;
        // 2. the single-image tile lists
        std::set<std::vector<int>> alone;
        for (int x = 0; x < G1; ++x) {
          std::vector<int> l;
          for (int t = x; t < j.ntiles; t += G1) l.push_back(t);
          alone.insert(l);
        }
        std::vector<int> cnt((size_t)total, 0);
        for (int x = 0; x < G; ++x) {
          std::vector<std::vector<int>> per(B);
          int prev_b = -1;
          for (int T = x; T < total; T += G) {
            const TileAt at = tile_at(j, T);
            const int t = at.y * j.tiles_x + at.x0 / j.tile_dx, b = at.b;
            if (b < 0 || b >= B || t < 0 || t >= j.ntiles || at.x0 % j.tile_dx) return fail(3, "layer %d: tile decode (image %d, tile %d)", r, b, t);
            if (b < prev_b) return fail(3, "layer %d: images out of order (image %d, tile %d)", r, b, t);
            prev_b = b;
            ++cnt[(size_t)b * j.ntiles + t];
            per[b].push_back(t);
            const int y = at.y, x0 = at.x0;
            // 3a. patch reads: the A operand (bulk copies) or the raw tensor normalised on load
            for (int g = 0; g < j.ngroups; ++g)
              for (int ri = 0; ri < j.nrows; ++ri)
                for (int cbi = 0; cbi < j.CbG; ++cbi) {
                  if (j.nl) {
                    const int ry = j.row_mul * y + j.grp_row[g][ri] - j.nl_padT, cb = j.grp_cb0[g] + cbi;
                    const int64_t row = ((int64_t)(ry >= 0 && ry < j.nl_H ? ry : 0) * j.nl_Cq + 2 * cb) * j.nl_Wp;
                    const int64_t lo4 = at.nl_raw4 + row, hi4 = at.nl_raw4 + row + j.nl_Wp + j.nl_Wp;
                    if (!Span{prev_raw.img / 4}.inside(b, lo4, hi4)) return fail(4, "layer %d: norm-on-load read outside image %d (tile %d)", r, b, t);
                    if (at.nl_sums + prev_stats < (int64_t)b * stats_img || at.nl_sums + prev_stats + 2 * j.nl_C > (int64_t)(b + 1) * stats_img)
                      return fail(4, "layer %d: norm-on-load statistics outside image %d (tile %d)", r, b, t);
                    continue;
                  }
                  for (int seg = 0; seg < j.nseg; ++seg) {
                    const int64_t s16 = ((int64_t)(j.row_mul * y + j.grp_row[g][ri]) * j.a_Cb + j.grp_cb0[g] + cbi) * j.a_slab16 +
                                        j.seg_src16[seg] + x0 + at.a16;
                    if (!Span{src.img16}.inside(b, s16, s16 + j.seg_len16[seg])) return fail(4, "layer %d: patch read outside image %d (tile %d)", r, b, t);
                  }
                }
            // 3b. the epilogue of each consumer thread (pixel r0 + 8h, channels c, c + 1)
            for (int th = 0; th < 256; ++th)
              for (int i = 0; i < j.Npad / 8; ++i)
                for (int h = 0; h < 2; ++h) {
                  if (j.opnd) {
                    int64_t o, so;
                    if (!opnd_epi_addr(j, T, th, i, h, o, so)) continue;
                    if (!Span{dst.img16 * 4}.inside(b, o, o + 1)) return fail(5, "layer %d: operand store outside image %d (tile %d)", r, b, t);
                    if (j.epi_skip && !Span{ops[block_in].img16 * 4}.inside(b, so, so + 1))
                      return fail(5, "layer %d: skip read outside image %d (tile %d)", r, b, t);
                    continue;
                  }
                  const int px = (th >> 7) * 64 + ((th >> 5) & 3) * 16 + ((th & 31) >> 2) + 8 * h, ch = 8 * i + 2 * (th & 3);
                  const int x = x0 + px;
                  if (j.xfold_kw) {  // x-fold: thread px < tile_dx stores every channel of pixel x0 + px
                    if (th >= j.tile_dx || x0 + th >= j.Wo || y >= j.Ho || i || h) continue;
                    const int xo = (x0 + th) * j.ox_mul + j.ox_off, yo = y * j.oy_mul + j.oy_off;
                    for (int k = 0; k < j.Cout; ++k) {
                      const int64_t o = at.out3 + (int64_t)k * j.Ho * j.Wo + (int64_t)yo * j.Wo + xo;
                      if (!Span{out_img}.inside(b, o, o + 1)) return fail(6, "layer %d: frame store outside image %d (tile %d)", r, b, t);
                    }
                    continue;
                  }
                  if (x >= j.Wo || y >= j.Ho || ch >= j.Cout) continue;
                  const int yo = y * j.oy_mul + j.oy_off, xo = x * j.ox_mul + j.ox_off;
                  if (last) {
                    for (int e = 0; e < 2; ++e) {
                      if (ch + e >= 3) continue;
                      const int64_t o = at.out3 + ((int64_t)(ch + e) * j.Ho + yo) * j.Wo + xo;
                      if (!Span{out_img}.inside(b, o, o + 1)) return fail(6, "layer %d: frame store outside image %d (tile %d)", r, b, t);
                    }
                    continue;
                  }
                  const int64_t o = at.raw + raw0 + (((int64_t)yo * j.raw_Cq + (ch >> 2)) * j.raw_Wp + xo) * 4 + (ch & 3);
                  if (!Span{raw.img}.inside(b, o, o + 2)) return fail(7, "layer %d: raw store outside image %d (tile %d)", r, b, t);
                  const int64_t s0 = at.stats + st0 + ch, s1 = at.stats + st0 + c.cout + ch;
                  if (!Span{stats_img}.inside(b, s0, s0 + 2) || !Span{stats_img}.inside(b, s1, s1 + 2))
                    return fail(8, "layer %d: statistics outside image %d (tile %d)", r, b, t);
                }
          }
          for (int b = 0; b < B; ++b)
            if (!per[b].empty() && !alone.count(per[b]))
              return fail(9, "layer %d: CTA tiles of image %d (first tile %d) are no single-image CTA's tiles", r, b, per[b][0]);
        }
        for (int T = 0; T < total; ++T)
          if (cnt[T] != 1) return fail(10, "layer %d: image %d tile %d not run exactly once", r, T / j.ntiles, T % j.ntiles);
      }
    }
    if (last) break;
    ops.push_back(dst);
    cur = (int)ops.size() - 1;
    prev_raw = raw;
    prev_stats = stats_off;
    if (!bn) stats_off += 2 * c.cout;
  }
  return 0;
}
