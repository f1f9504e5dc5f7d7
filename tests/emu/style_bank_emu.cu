// style_bank_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of how conv_tc_kernel's batched instances pick each image's style
// (ConvJob::img_style, fav_net_add_style) over every convolution of a net's plan.  The jobs come from the product's planner
// (conv_plan.hpp) and its slot chooser (conv_tc_choose_slots); the per-image parameters from the helper the kernel calls
// (style_at, conv.cuh), on host banks whose every entry names its style.  Not part of libfav_b200.so.
#include "conv_emu.cu"

namespace {
int failf(int code, const char *what, int layer, int cta, int tile) {
  set_error("layer %d, CTA %d, tile %d: %s", layer, cta, tile, what);
  return code;
}
// a parameter buffer's per-style stride as net.cu's dev_upload rounds it (bytes up to a multiple of 256)
int64_t bank_stride(int64_t bytes, int elem) { return (std::max<int64_t>(bytes, 16) + 255) / 256 * 256 / elem; }
}  // namespace

// rows: n x 8 ints as emu_batch_check reads them (batch_emu.cu): {type, cin, cout, k, stride, pad, transposed, adj}, type 0 =
// conv, 1 = nearest upsampling by `stride`, 2 = first conv of an R/C block, 3 = second conv of an R block, 4 = second conv of a
// C block; the last row is the final convolution.  bn: batch-normalized net (operand epilogues); else InstanceNorm, with
// norm-on-load where net.cu fuses it (a conv whose input norm adds no skip, whose patch the producers can fill).  in_H / in_W:
// the net input including the reflection padding.  styles[b] in [0, S): the style of image b of a batch of B on num_sms
// persistent CTAs; single: the single-pass instances (ConvJob::single).  For every tensor-core job, each role's walk of its
// CTA's tiles, as conv_tc.cu runs it, is checked:
//   1. consumers: each image's tiles take the bias, 2^-w_exp and (operand epilogue) scale of that image's style;
//   2. weight producer: every chunk the consumers read for a tile comes from that tile's style, inside that style's packed
//      weights (resident weights: the chunks of the CTA's first tile), and announces (FAV_TC_B_CHUNK_TX) exactly the bytes it
//      copies.  Residency as the product decides it (tc_may_keep_weights); allow_resident = 1 keeps every job that fits
//      resident, as a net with one style does, to show that check 2 fails on it;
//   3. norm-on-load producers: the table each tile normalises with holds its image's style's gamma and beta;
//   4. patch producer: the bytes it announces (tc_a_stage_tx) equal the bytes its copies bring.
// info[5]: jobs, jobs normalising on load, jobs with an operand epilogue, style changes along CTA tile sequences, resident jobs.
extern "C" int emu_style_bank_check(int n, const int *rows, int in_H, int in_W, int bn, int B, const int *styles, int S,
                                    int num_sms, int single, int allow_resident, int *info) {
  for (int b = 0; b < B; ++b)
    if (styles[b] < 0 || styles[b] >= S) { set_error("style %d of image %d out of range", styles[b], b); return 1; }
  std::vector<ConvDef> convs(n);
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) continue;
    init_conv_def(convs[r], "l" + std::to_string(r), d[1], d[2], d[3], d[4], d[5], d[6] != 0, d[7]);
    build_phases(convs[r]);
    convs[r].raw_out = r + 1 < n;
    if (plan_conv_nblocks(convs[r]) != FAV_OK) return 1;
    if (!bn && plan_phase_stack(convs[r]) != FAV_OK) return 1;
  }
  auto next_conv = [&](int r) -> const ConvDef * {
    for (int q = r + 1; q < n; ++q)
      if (rows[8 * q] != 1) return &convs[q];
    return nullptr;
  };
  for (int i = 0; i < 5; ++i) info[i] = 0;
  std::vector<float> unscale(S);
  for (int s = 0; s < S; ++s) unscale[s] = ldexpf(1.f, -1 - s);  // a distinct 2^-w_exp per style
  Operand cur = operand_geometry(rows[1], in_H, in_W, next_conv(-1));
  cur.img16 = (int64_t)cur.elems16;
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) {
      cur = operand_geometry(cur.C, cur.H * d[4], cur.W * d[4], next_conv(r));
      cur.img16 = (int64_t)cur.elems16;
      continue;
    }
    const ConvDef &c = convs[r];
    const bool last = r + 1 == n;
    const bool try_nl = !bn && r > 0 && rows[8 * (r - 1)] != 1 && rows[8 * (r - 1)] != 3 && d[0] != 2 && c.cin <= 256;
    int ho, wo;
    conv_out_size(c, cur.H, cur.W, &ho, &wo);
    Operand dst = operand_geometry(c.cout, ho, wo, last ? nullptr : next_conv(r));
    dst.img16 = (int64_t)dst.elems16;
    const int nb = c.nblock.empty() ? 1 : (int)c.nblock.size();
    const bool stack = !c.stack.empty();
    for (int blk = 0; blk < nb; ++blk) {
      const ConvDef &cd = c.nblock.empty() ? c : c.nblock[blk];
      for (const ConvPhase &ph : stack ? c.stack : cd.phases) {
        ConvJob j;
        if (fill_conv_job(cd, ph, cur, j) != FAV_OK) return 2;
        set_conv_batch(j, B, 0, 3ll * in_H * in_W, 1);
        j.final_mode = last ? 1 : 0;
        j.single = single;
        // the banks: entry i of style s of every buffer holds s (weights: the tag {s, i}), bias c of style s is 4096 s + c
        const int64_t npk16 = (int64_t)j.ngroups * j.nchunks * j.chunk16, wstride = bank_stride(npk16 * 16, 16);
        std::vector<uint4> wbank((size_t)S * wstride);
        for (int s = 0; s < S; ++s)
          for (int64_t i = 0; i < wstride; ++i) wbank[(size_t)(s * wstride + i)] = make_uint4((unsigned)s, (unsigned)i, 0x5151u, (unsigned)r);
        const int64_t pstride = bank_stride((int64_t)j.Npad * 4, 4);
        std::vector<float> bias((size_t)S * pstride), scale((size_t)S * pstride);
        for (int s = 0; s < S; ++s)
          for (int64_t i = 0; i < pstride; ++i) { bias[(size_t)(s * pstride + i)] = 4096.f * s + i; scale[(size_t)(s * pstride + i)] = -4096.f * s - i; }
        j.b = wbank.data(); j.bias = bias.data();
        if (!last && bn) set_opnd_epilogue(j, blk, scale.data(), dst, 1, nullptr, 0);
        const int64_t nstride = bank_stride((int64_t)c.cin * 4, 4);
        std::vector<float> gamma((size_t)S * nstride), beta((size_t)S * nstride);
        for (int s = 0; s < S; ++s)
          for (int64_t i = 0; i < nstride; ++i) { gamma[(size_t)(s * nstride + i)] = 4096.f * s + i; beta[(size_t)(s * nstride + i)] = -4096.f * s - i; }
        // net.cu set_job_styles / fuse_norm_on_load
        j.img_style = styles; j.w_unscale_style = unscale.data(); j.b_style16 = wstride; j.bias_style = (int)pstride;
        if (try_nl && nl_geometry_ok(j) && !j.xfold_kw) {
          j.nl = 1; j.nl_gamma = gamma.data(); j.nl_beta = beta.data(); j.nl_C = c.cin; j.nl_style = (int)nstride;
        }
        conv_tc_choose_slots(j);  // this emulator's copy of the slot chooser (conv_emu.cu), whose residency ignores styles
        if (j.b_resident && !allow_resident && !tc_may_keep_weights(j)) { j.b_resident = 0; j.b_slots = std::max(j.b_slots, 2); }
        if (j.b_resident) ++info[4];
        if (!j.b_resident && j.b_slots < 2) return failf(3, "weight ring below two slots", r, 0, 0);
        if (conv_tc_smem_bytes(j) > 227 * 1024) return failf(3, "shared memory budget exceeded", r, 0, 0);
        ++info[0];
        info[1] += j.nl;
        info[2] += j.opnd;
        const bool pair = !j.single;
        const int total = B * j.ntiles, G = std::min(total, num_sms);
        for (int x = 0; x < G; ++x) {
          // 1. consumers (tc_consume): per image of the CTA, its style's bias / 2^-w_exp / epilogue scale
          for (int tile = x; tile < total;) {
            const TileAt img = tile_at(j, tile);
            const int img_end = std::min(total, (img.b + 1) * j.ntiles), s = styles[img.b];
            const StyleAt sty = style_at(j, img.b);
            for (; tile < img_end; tile += G) {
              if (tile_at(j, tile).b != img.b) return failf(4, "consumer tile of another image", r, x, tile);
              for (int ch = 0; ch < j.Npad; ch += 2)
                if (sty.bias[ch] != 4096.f * s + ch || sty.bias[ch + 1] != 4096.f * s + ch + 1)
                  return failf(4, "consumer bias of another style", r, x, tile);
              if (sty.w_unscale != unscale[s]) return failf(4, "consumer 2^-w_exp of another style", r, x, tile);
              if (j.opnd && sty.epi_scale[j.Npad - 1] != -4096.f * s - (j.Npad - 1)) return failf(4, "epilogue scale of another style", r, x, tile);
            }
          }
          // 2. weight producer: the chunks of each tile from its image's style, the bytes announced = the bytes copied.  The
          // consumers of a resident job read the chunks its first tile loaded
          int prev_s = -1;
          for (int tile = x; tile < total; tile += G) {
            const int s = styles[tile_at(j, tile).b];
            if (prev_s >= 0 && s != prev_s) ++info[3];
            prev_s = s;
            const uint4 *wb = style_at(j, tile_at(j, j.b_resident ? x : tile).b).b;
            for (int g = 0; g < j.ngroups; ++g)
              for (int ch = 0; ch < j.nchunks; ++ch) {
                const uint32_t tx = FAV_TC_B_CHUNK_TX(j.dbg, (uint32_t)j.chunk16 * 16u, pair);
                const int64_t i0 = (int64_t)(g * j.nchunks + ch) * j.chunk16, len16 = (pair ? j.chunk16 : j.chunk16 / 2);
                const uint4 *src = wb + i0;
                if (src < wbank.data() + (int64_t)s * wstride || src + len16 > wbank.data() + (int64_t)s * wstride + npk16)
                  return failf(5, "weight chunk outside its style's packed weights", r, x, tile);
                if ((int64_t)tx != len16 * 16) return failf(5, "weight bytes announced differ from those copied", r, x, tile);
                for (const uint4 *p : {src, src + len16 - 1})
                  if (p->x != (unsigned)s || p->y != (unsigned)(p - wbank.data() - (int64_t)s * wstride))
                    return failf(5, "weight chunk of another style", r, x, tile);
              }
          }
          // 3. norm-on-load producers: the table of the tile's image's style, rebuilt when the image changes
          if (j.nl) {
            int nl_b = x / j.ntiles;
            std::vector<float> tab_g(c.cin), tab_b(c.cin);
            auto build = [&](int b) {
              const StyleAt sty = style_at(j, b);
              for (int ci = 0; ci < c.cin; ++ci) { tab_g[ci] = sty.nl_gamma[ci]; tab_b[ci] = sty.nl_beta[ci]; }
            };
            build(nl_b);
            for (int tile = x; tile < total; tile += G) {
              const TileAt at = tile_at(j, tile);
              if (at.b != nl_b) { nl_b = at.b; build(nl_b); }
              const int s = styles[at.b];
              for (int ci = 0; ci < c.cin; ++ci)
                if (tab_g[ci] != 4096.f * s + ci || tab_b[ci] != -4096.f * s - ci) return failf(6, "norm table of another style", r, x, tile);
            }
          } else {
            // 4. patch producer: one stage's copies as conv_tc.cu issues them
            const int NP = pair ? 2 : 1, per_row = j.CbG * j.nseg * NP, ncopies = j.nrows * per_row;
            uint64_t copied = 0;
            for (int cp = 0; cp < ncopies; ++cp) {
              int rr = cp % per_row;
              rr -= rr / (j.nseg * NP) * j.nseg * NP;
              copied += (uint64_t)((j.dbg & 4) ? 1 : j.seg_len16[pair ? rr >> 1 : rr]) * 16u;
            }
            if (copied != tc_a_stage_tx(j, pair)) return failf(7, "patch bytes announced differ from those copied", r, x, 0);
          }
        }
      }
    }
    if (last) break;
    cur = dst;
  }
  return 0;
}
