// arena_emu.cu -- TEST INFRASTRUCTURE: the stylization net's operands and steps as net.cu's build_plan lays them out (operand
// geometries from operand_geometry), placed in one arena by the product's planner (plan_arena, arena_plan.hpp), then the frame
// replayed on a byte-ownership map of the arena.  Not part of libfav_b200.so.
#include "conv_emu.cu"
#include "../../fast-artistic-videos_b200/csrc/arena_plan.hpp"

namespace {
int fail(const char *fmt, int a, int b) {
  char buf[256];
  snprintf(buf, sizeof(buf), fmt, a, b);
  set_error("%s", buf);
  return 1;
}
}  // namespace

// rows: as emu_batch_check (batch_emu.cu) reads them.  bn: a batch-normalized net, whose conv epilogue writes the next operand
// and reads the skip.  in_H / in_W: the net input including the reflection padding.  Checked, for a batch of B images:
//   1. no two operands whose lifetimes overlap share a byte;
//   2. every operand a step reads was written by an earlier step (the first operand: before the steps) and no operand written
//      since has taken over any of its bytes;
//   3. the operands plan_arena reports kept are exactly those whose bytes no later operand took over.
// out[4]: all-live bytes of the operands in the arena, arena bytes, operands, operands kept.
extern "C" int emu_arena_check(int n, const int *rows, int in_H, int in_W, int bn, int B, int64_t *out) {
  std::vector<ConvDef> convs(n);
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) continue;
    init_conv_def(convs[r], "l" + std::to_string(r), d[1], d[2], d[3], d[4], d[5], d[6] != 0, d[7]);
    build_phases(convs[r]);
  }
  auto next_conv = [&](int r) -> const ConvDef * {
    for (int q = r + 1; q < n; ++q)
      if (rows[8 * q] != 1) return &convs[q];
    return nullptr;
  };
  // build_plan's operands and steps: UX -> one upsampling step; a conv -> the conv step, then (not the last) its norm step
  std::vector<Operand> ops;
  std::vector<ArenaStep> steps;
  ops.push_back(operand_geometry(rows[1], in_H, in_W, next_conv(-1)));
  int cur = 0, block_in = -1;
  for (int r = 0; r < n; ++r) {
    const int *d = rows + 8 * r;
    if (d[0] == 1) {
      ops.push_back(operand_geometry(ops[cur].C, ops[cur].H * d[4], ops[cur].W * d[4], next_conv(r)));
      ArenaStep s;
      s.src = cur; s.dst = cur = (int)ops.size() - 1;
      steps.push_back(s);
      continue;
    }
    if (d[0] == 2) block_in = cur;
    int ho, wo;
    conv_out_size(convs[r], ops[cur].H, ops[cur].W, &ho, &wo);
    ArenaStep cs, ns;
    cs.src = cur;
    if (r + 1 == n) { steps.push_back(cs); break; }
    ops.push_back(operand_geometry(d[2], ho, wo, next_conv(r)));
    ns.dst = cur = (int)ops.size() - 1;
    ns.skip = d[0] == 3 ? block_in : -1;
    if (bn) { cs.dst = ns.dst; cs.skip = ns.skip; }
    steps.push_back(cs);
    steps.push_back(ns);
  }
  const int nop = (int)ops.size();
  std::vector<size_t> bytes(nop);
  std::vector<char> pinned(nop, 0);
  for (int i = 0; i < nop; ++i) bytes[i] = 2 * (((size_t)B * ops[i].elems16 * 16 + kArenaAlign - 1) / kArenaAlign * kArenaAlign);
  pinned[0] = 1;
  const ArenaPlan p = plan_arena(steps, bytes, pinned);
  auto overlap = [&](int i, int j) { return p.off[i] < p.off[j] + bytes[j] && p.off[j] < p.off[i] + bytes[i]; };
  // 1.
  for (int i = 1; i < nop; ++i) {
    if (p.first[i] < 0) return fail("operand %d is never written (%d)", i, 0);
    if (p.off[i] % kArenaAlign || p.off[i] + bytes[i] > p.arena_bytes) return fail("operand %d outside the arena (%d)", i, 0);
    for (int j = 1; j < i; ++j)
      if (p.first[i] <= p.last[j] && p.first[j] <= p.last[i] && overlap(i, j)) return fail("live operands %d and %d share bytes", i, j);
  }
  // 2. and 3.: replay the frame; an operand written at step s takes its bytes over from every operand holding any of them
  std::vector<char> written(nop, 0), lost(nop, 0);
  written[0] = 1;
  for (int s = 0; s < (int)steps.size(); ++s) {
    for (int r : {steps[s].src, steps[s].skip}) {
      if (r < 0) continue;
      if (!written[r]) return fail("step %d reads operand %d before it is written", s, r);
      if (lost[r]) return fail("step %d reads operand %d after a later operand took its bytes", s, r);
    }
    const int w = steps[s].dst;
    if (w >= 0 && !written[w]) {
      for (int j = 1; j < nop; ++j)
        if (j != w && written[j] && overlap(w, j)) lost[j] = 1;
      written[w] = 1;
    }
  }
  int kept = 0;
  for (int i = 1; i < nop; ++i) {
    if ((p.kept[i] != 0) != !lost[i]) return fail("operand %d: kept flag %d disagrees with the replay", i, p.kept[i]);
    kept += p.kept[i] != 0;
  }
  out[0] = (int64_t)p.all_live_bytes; out[1] = (int64_t)p.arena_bytes; out[2] = nop; out[3] = kept;
  return 0;
}
