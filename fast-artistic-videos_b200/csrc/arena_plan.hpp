// arena_plan.hpp -- host-only buffer planner of the stylization net's activation operands: one arena in which operands whose
// lifetimes do not overlap share bytes.  Pure functions, so the same code runs on the CPU in tests/emu/arena_emu.cu and in
// net.cu's build_plan.
//
// A frame's steps run in order on one stream.  Operand i is live from the step that writes it (first[i]) to the last step
// that reads it (last[i]): as a convolution's A operand, as the skip of a residual block, or as the operand a conv normalises
// on load stands for.  Two operands may share bytes only when one's last step comes before the other's first.  Kernels
// write only an operand's interior pixels, so an operand that takes over bytes finds its previous occupant's data in its
// zero border and slack: net.cu clears them (launch_clear_border) right before the step that writes it.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace fav {

// one step of a plan as the planner sees it: the operand it writes and the operands it reads (-1: none)
struct ArenaStep {
  int dst = -1;
  int src = -1, skip = -1;
};

struct ArenaPlan {
  std::vector<int> first, last;  // per operand: the step that writes it, the last step that reads it (-1: pinned)
  std::vector<size_t> bytes;     // per operand, as given
  std::vector<size_t> off;       // byte offset in the arena (pinned operands: unused)
  std::vector<char> kept;        // its bytes are intact after the last step (no later operand takes any of them over)
  size_t arena_bytes = 0;        // size of the arena
  size_t all_live_bytes = 0;     // the same operands, each in its own buffer
};

constexpr size_t kArenaAlign = 256;  // cudaMalloc's alignment: every operand keeps the alignment of its own buffer

// bytes[i]: operand i's size; pinned[i]: operand i keeps its own buffer (it is written or read outside the step list).
// Greedy first-fit, largest operand first: each operand goes to the lowest offset at which it overlaps no operand placed
// before it whose lifetime overlaps its own.
static inline ArenaPlan plan_arena(const std::vector<ArenaStep> &steps, const std::vector<size_t> &bytes,
                                   const std::vector<char> &pinned) {
  const int n = (int)bytes.size();
  ArenaPlan p;
  p.bytes = bytes;
  p.first.assign(n, -1); p.last.assign(n, -1); p.off.assign(n, 0); p.kept.assign(n, 1);
  for (int s = 0; s < (int)steps.size(); ++s) {
    const ArenaStep &st = steps[s];
    if (st.dst >= 0 && p.first[st.dst] < 0) p.first[st.dst] = s;
    for (int r : {st.src, st.skip})
      if (r >= 0) p.last[r] = std::max(p.last[r], s);
  }
  std::vector<int> order;
  for (int i = 0; i < n; ++i) {
    if (pinned[i] || p.first[i] < 0) { p.first[i] = p.last[i] = -1; continue; }
    p.last[i] = std::max(p.last[i], p.first[i]);
    p.all_live_bytes += bytes[i];
    order.push_back(i);
  }
  auto size_of = [&](int i) { return (bytes[i] + kArenaAlign - 1) / kArenaAlign * kArenaAlign; };
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return size_of(a) > size_of(b); });
  std::vector<int> placed;
  for (int i : order) {
    std::vector<std::pair<size_t, size_t>> busy;  // [begin, end) of placed operands live at the same time
    for (int j : placed)
      if (p.first[j] <= p.last[i] && p.first[i] <= p.last[j]) busy.push_back({p.off[j], p.off[j] + size_of(j)});
    std::sort(busy.begin(), busy.end());
    size_t at = 0;
    for (const auto &b : busy) {
      if (at + size_of(i) <= b.first) break;
      at = std::max(at, b.second);
    }
    p.off[i] = at;
    p.arena_bytes = std::max(p.arena_bytes, at + size_of(i));
    placed.push_back(i);
  }
  for (int i : order)
    for (int j : order)
      if (p.first[j] > p.first[i] && p.off[j] < p.off[i] + bytes[i] && p.off[i] < p.off[j] + bytes[j]) p.kept[i] = 0;
  return p;
}

}  // namespace fav
