// opnd_epi_emu.cu -- TEST INFRASTRUCTURE: CPU emulation of conv_tc_kernel's operand epilogue (batch-normalized nets, ConvJob::opnd)
// over every non-final convolution of a net's plan.  The jobs come from the product's planner (plan_conv_nblocks,
// operand_geometry, fill_conv_job, set_opnd_epilogue in conv_plan.hpp) and the stores from the address helper the kernel
// itself calls (opnd_epi_addr, conv.cuh).  Not part of libfav_b200.so.
#include "conv_emu.cu"

// storage coordinates of a 4-byte word of operand o, decoded independently of Operand::off16
static void decode_word(const Operand &o, int64_t w, int *ys, int *xs, int *c) {
  const int64_t u = w / 4, slab = o.slab16();
  const int64_t in = u % slab, rest = u / slab;
  *xs = (int)(o.parity ? (in < o.Ws2 ? 2 * in : 2 * (in - o.Ws2) + 1) : in);
  *c = (int)(rest % o.Cb) * 8 + (int)(w % 4) * 2;
  *ys = (int)(rest / o.Cb);
}

// rows: n x 8 ints {type, cin, cout, k, stride, pad, transposed, adj} in execution order, as net.cu's fav_net_create lays a net
// out: type 0 = conv (+BN +ReLU), 1 = nearest upsampling by `stride` (its BN stays a separate pass), 2 = first conv of an R/C
// block, 3 = second conv of an R block (skip from the block input), 4 = second conv of a C block (ReLU, no skip).  The last row
// is the final convolution, which keeps its tanh epilogue.  in_H / in_W: the net input including the reflection padding.
// Every non-final convolution writes its consumer's operand through opnd_epi_addr; checked: every interior (pixel, channel
// pair) of that operand is written exactly once, nothing in its zero border / slack / padding channels, every residual skip
// read is the interior pixel `shave` further in the block input.  info[4]: jobs, jobs with a parity-split destination, jobs of
// transposed-conv phases (oy_mul 2), jobs of N blocks past the first.
extern "C" int emu_opnd_epi_check(int n, const int *rows, int in_H, int in_W, int *info) {
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
  std::vector<Operand> ops;
  ops.push_back(operand_geometry(rows[1], in_H, in_W, next_conv(-1)));
  int cur = 0, block_in = -1;
  for (int r = 0; r + 1 < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) {
      ops.push_back(operand_geometry(ops[cur].C, ops[cur].H * d[4], ops[cur].W * d[4], next_conv(r)));
      cur = (int)ops.size() - 1;
      continue;
    }
    const ConvDef &c = convs[r];
    if (d[0] == 2) block_in = cur;
    int ho, wo;
    conv_out_size(c, ops[cur].H, ops[cur].W, &ho, &wo);
    ops.push_back(operand_geometry(c.cout, ho, wo, next_conv(r)));
    const Operand dst = ops.back(), src = ops[cur];
    const bool skip = d[0] == 3;
    const Operand *sk = skip ? &ops[block_in] : nullptr;
    const int shave = c.pad == 0 ? 2 : 0;  // ShaveImage(2) ('reflect-start', pad-0 block convs) or Identity ('zero')
    std::vector<uint8_t> cnt(dst.elems16 * 4, 0);
    const int nb = c.nblock.empty() ? 1 : (int)c.nblock.size();
    for (int b = 0; b < nb; ++b) {
      const ConvDef &cd = c.nblock.empty() ? c : c.nblock[b];
      for (const ConvPhase &ph : cd.phases) {
        ConvJob j;
        if (fill_conv_job(cd, ph, src, j) != FAV_OK) return 2;
        set_opnd_epilogue(j, b, nullptr, dst, d[0] != 3, sk, shave);
        ++info[0];
        info[1] += dst.parity;
        info[2] += j.oy_mul == 2;
        info[3] += b > 0;
        for (int tile = 0; tile < j.ntiles; ++tile)
          for (int t = 0; t < 256; ++t)
            for (int i = 0; i < j.Npad / 8; ++i)
              for (int h = 0; h < 2; ++h) {
                int64_t o, so;
                if (!opnd_epi_addr(j, tile, t, i, h, o, so)) continue;
                if (o < 0 || o >= (int64_t)cnt.size()) { set_error("layer %d: store outside the operand", r); return 3; }
                if (cnt[o] < 255) ++cnt[o];
                int ys, xs, ch;
                decode_word(dst, o, &ys, &xs, &ch);
                if (skip) {
                  if (so < 0 || so >= (int64_t)sk->elems16 * 4) { set_error("layer %d: skip read outside the block input", r); return 4; }
                  int sy, sx, sc;
                  decode_word(*sk, so, &sy, &sx, &sc);
                  if (sy - sk->padT != ys - dst.padT + shave || sx - sk->padL != xs - dst.padL + shave || sc != ch ||
                      sy < sk->padT || sy >= sk->padT + sk->H || sx < sk->padL || sx >= sk->padL + sk->W) {
                    set_error("layer %d: skip read at (%d,%d,c%d) for output (%d,%d,c%d)", r, sy, sx, sc, ys, xs, ch);
                    return 4;
                  }
                }
              }
      }
    }
    for (int64_t w = 0; w < (int64_t)cnt.size(); ++w) {
      int ys, xs, ch;
      decode_word(dst, w, &ys, &xs, &ch);
      const bool interior = ys >= dst.padT && ys < dst.padT + dst.H && xs >= dst.padL && xs < dst.padL + dst.W && ch < dst.C;
      if (cnt[w] != (interior ? 1 : 0)) {
        set_error("layer %d: word %lld (row %d, x %d, channel %d, %s) written %d times", r, (long long)w, ys, xs, ch,
                  interior ? "interior" : "border / slack", (int)cnt[w]);
        return 5;
      }
    }
    cur = (int)ops.size() - 1;
  }
  return 0;
}
