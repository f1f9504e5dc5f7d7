// avg_emu.cu -- TEST INFRASTRUCTURE: the exact parallel CMatrix::avg of consistency.cu run on the host.  The sub-chunk and
// chunk records, the estimate that picks the hypotheses and the combine walk use the helpers of exact_avg.cuh that the kernels
// (avg_sum_kernel, avg_hyp_kernel, avg_walk_kernel) use; the reference is the plain sequential loop (emu_avg_seq).  Built with
// -ffp-contract=off.  Not part of libfav_b200.so.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../fast-artistic-videos_b200/csrc/exact_avg.cuh"

using namespace fav;

extern "C" float emu_avg_seq(const float *x, int64_t n) {
  float a = 0.f;
  for (int64_t i = 0; i < n; ++i) a = a + x[i];
  return a / (float)(int)n;
}

// stats[3]: chunks that jumped, sub-chunks that jumped, sub-chunks run as FADDs
extern "C" float emu_avg_exact(const float *x, int64_t n, int64_t *stats) {
  const int64_t nsub = (n + kAvgSub - 1) / kAvgSub, nch = (nsub + kAvgGroup - 1) / kAvgGroup;
  std::vector<double> ssum(nsub, 0.0), csum(nch, 0.0);
  for (int64_t s = 0; s < nsub; ++s) {
    for (int64_t e = s * kAvgSub; e < std::min(n, (s + 1) * kAvgSub); ++e) ssum[s] += x[e];
    csum[s / kAvgGroup] += ssum[s];
  }
  std::vector<AvgRec> srec(nsub), crec(nch);
  double S = 0.0;
  for (int64_t c = 0; c < nch; ++c) {
    const int64_t s0 = c * kAvgGroup;
    const int ns = (int)std::min<int64_t>(kAvgGroup, nsub - s0);
    crec[c].ebase = avg_estimate_exp(S);
    double sp = S;
    for (int g = 0; g < ns; ++g) {
      const int64_t e0 = (s0 + g) * kAvgSub;
      srec[s0 + g].ebase = avg_sub_ebase(crec[c].ebase, sp);
      sp += ssum[s0 + g];
      for (int h = 0; h < kAvgHyps; ++h)
        srec[s0 + g].h[h] = avg_simulate_hyp(x + e0, (int)std::min<int64_t>(kAvgSub, n - e0), srec[s0 + g].ebase, h);
    }
    for (int h = 0; h < kAvgHyps; ++h) {
      AvgHyp acc = srec[s0].h[h];
      for (int g = 1; g < ns; ++g) acc = avg_compose(acc, h & 1, srec[s0 + g].h[h & ~1], srec[s0 + g].h[h | 1]);
      crec[c].h[h] = acc;
    }
    S += csum[c];
  }
  stats[0] = stats[1] = stats[2] = 0;
  float a = 0.f;
  for (int64_t c = 0; c < nch; ++c) {
    float j;
    if (avg_try_jump(a, crec[c], &j)) { a = j; ++stats[0]; continue; }
    const int64_t s0 = c * kAvgGroup;
    for (int64_t s = s0; s < std::min(nsub, s0 + kAvgGroup); ++s) {
      if (avg_try_jump(a, srec[s], &j)) { a = j; ++stats[1]; continue; }
      ++stats[2];
      for (int64_t e = s * kAvgSub; e < std::min(n, (s + 1) * kAvgSub); ++e) a = avg_fadd(a, x[e]);
    }
  }
  return avg_finish(a, n);
}

extern "C" int emu_avg_sub() { return kAvgSub; }
extern "C" int emu_avg_chunk() { return kAvgChunk; }
