// net.cu -- host side of the stylization network: arch parser, parameter store, weight repacking, per-size
// execution plan, forward, run_image / run_next_image.
//   models_video.build_model              fast_artistic_video/models_video.lua:55-140
//   build_res_block (reflect-start)       models_video.lua:41-53
//   lazily inserted reflection padding    train_video.lua:316-325
//   run_image / run_next_image            fast_artistic_video_core.lua:121-180
#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>
#include <cmath>
#include <cstring>

#include "arena_plan.hpp"
#include "conv_plan.hpp"

namespace fav {

int launch_temporal_input(const float *content, const float *prev, const float *flow, const float *cert,
                          const float *fill, const float *flow_mask, float *out7, int H, int W, int border_mode,
                          bool first, cudaStream_t st, int nimg = 1);
int launch_temporal_stage(const float *content, const float *prev, const float *flow, const float *fw_uv, const float *cert_raw,
                          const float *fill, const float *flow_mask, float *out7, float *cert_out, const Operand *dst, int R,
                          int H, int W, int r, int border_mode, cudaStream_t st, int nimg = 1);
int launch_min_filter(const float *in, float *out, int n, int H, int W, int r, cudaStream_t st);
int launch_consistency(const float *f1u, const float *f1v, const float *f2u, const float *f2v, const float *structure,
                       const float *avg_dev, float avg_host, uint8_t *rel, float *cert, int W, int H, cudaStream_t st);
int launch_temporal_input_packed(const float *content, const float *prev, const float *flow, const float *cert,
                                 const float *fill, const float *flow_mask, const Operand &dst, int R, int H, int W,
                                 int border_mode, bool first, cudaStream_t st, int nimg = 1);
int launch_temporal_stage_structure(const float *content, const float *prev, const float *flow, const float *fw_uv,
                                    const float *structure, const float *structure_avg, const float *fill, const float *flow_mask,
                                    float *cert_out, const Operand &dst, int R, int H, int W, int r, int border_mode, cudaStream_t st);
int launch_compute_corners(const float *image, float scale, int Z, int W, int H, float rho, float *corners, float *avg_out,
                           void *workspace, cudaStream_t st);
int launch_clear_border(const Operand &o, int nimg, cudaStream_t st);
int launch_image_scale_bicubic(const float *in, float *out, int C, int Hin, int Win, int Hout, int Wout, cudaStream_t st);
int check_scale_args(const float *in, const float *out, int C, int Hin, int Win, int Hout, int Wout);

// ---------------------------------------------------------------------------------------------------------
struct Param {
  std::string name;
  int64_t shape[4] = {1, 1, 1, 1};
  int64_t numel = 0;
  std::vector<float> host;
  bool set = false;
};

// a normalisation layer: InstanceNormalization, or (batch-normalized nets) inference-mode SpatialBatchNormalization
struct InDef {
  std::string name;
  int C = 0;
  float *d_gamma = nullptr, *d_beta = nullptr;
  int pw = -1, pb = -1;
  // batch norm: running statistics and eps; conv = the convolution it directly follows (folded into it at finalize,
  // fold_batch_norms), -1 after a UX upsampling (applied as the fixed per-channel affine d_mean / d_scale by up_apply)
  int pm = -1, pv = -1, pe = -1, conv = -1;
  std::vector<float> h_mean, h_scale;
  float *d_mean = nullptr, *d_scale = nullptr;
};

// arch-level program
struct SpecOp {
  int kind;  // 0 conv(+in+relu), 1 conv block: two 3x3 convs + IN (RX: + ShaveImage / Identity skip; CX: no skip, ReLU after),
             // 2 nearest upsampling (+in+relu)
  bool skip = true;   // kind 1: residual (RX) or plain (CX) block
  int shave = 2;      // kind 1: ShaveImage(2) ('reflect-start') or Identity ('zero') on the skip branch
  int scale = 1;
  int conv[2] = {-1, -1};
  int inorm[2] = {-1, -1};
  bool relu = false, last = false;
};

struct PlanStep {
  int kind;  // 0 conv, 1 instance norm (+relu, +skip) -> operand, 2 nearest upsampling + instance norm + relu
  int scale = 1;
  int conv = -1, inorm = -1;
  int src = -1, dst = -1, skip = -1;
  int relu = 0;
  int shave = 2;
  RawTensor raw;
  std::vector<ConvJob> tc;
  std::vector<ConvJob> tc_plain;  // kind 0 normalising on load: the same jobs reading the in_apply'd operand (replay_unfused)
  std::vector<SimtJob> simt;
  int stats_off = 0;
  int raw_sel = 0;       // raw.p is Plan::raw_buf (0) or raw_buf2 (1)
  int layer_index = -1;  // arch token index whose output this step completes (for fav_net_layer_output)
  bool fused_nl = false; // kind 1: the tensor-core consumer normalises on load (conv_tc.cu), this pass is skipped
  int clear = -1;        // arena plans: the operand this step writes first, whose border it zeroes before it runs
};

// a batch: B frames of one size run through one plan, every kernel covering all B images in one launch (conv.cuh tile_at);
// operands, raw tensors and statistics hold one image after the other, each with its own zero border
constexpr int kMaxBatch = 64;
constexpr size_t kMaxPlanBytes = (size_t)32 << 30;  // default activation budget of one plan (fav_net_set_activation_budget)

struct Plan {
  int B = 1, H = 0, W = 0;
  size_t bytes = 0;        // device memory of the activation buffers, checked against budget before each allocation
  size_t budget = kMaxPlanBytes;
  bool dry = false;        // sizes only: alloc_zero counts bytes and allocates nothing (build_plan's first pass)
  // arena plan (arena_plan.hpp): operands share one buffer by lifetime.  preset: the hi / lo pointers make_operand hands out
  // (null: its own buffer); kept: per operand, whether its bytes are intact after the frame (fav_net_layer_output)
  void *arena = nullptr;
  std::vector<std::pair<__half *, __half *>> preset;
  std::vector<char> kept;
  int64_t stats_img = 0;   // doubles of statistics per image
  std::vector<Operand> ops;
  std::vector<void *> allocs;
  float *raw_buf = nullptr, *raw_buf2 = nullptr;  // consecutive convolutions alternate (norm-on-load reads one, writes the other)
  size_t raw_bytes = 0;  // of each; a batch-normalized net allocates them only for the CUDA-core comparator (ensure_raw)
  double *stats = nullptr;
  size_t stats_bytes = 0;  // all B images
  float *msb = nullptr;
  float *in7 = nullptr, *out3 = nullptr;  // scratch for run_image / run_next_image
  float *cert_a = nullptr, *cert_b = nullptr;  // scratch of the unfused fallback of fav_run_next_image_flows
  // 4-argument mode (fav_run_next_image_flows_structure): the corners plane, its average and fav_compute_corners' workspace,
  // allocated on the first such call
  float *structure = nullptr, *structure_avg = nullptr;
  void *corners_ws = nullptr;
  // -scale_factor (fav_run_image_scaled): the content resampled to this plan's size, allocated on the first such call
  float *scaled_in = nullptr;
  std::vector<PlanStep> steps;
  // a net with a style bank (fav_net_add_style): the style of each image, read by every batched kernel (ConvJob::img_style),
  // and the assignment it holds, which bind_styles rewrites on the call's stream when it changes; null with one style
  int *styles = nullptr;
  std::vector<int> styles_host;
  std::map<int, int> layer_operand;  // arch token index -> operand holding its output
  // CUDA graphs of the whole per-frame kernel sequence (run_[next_]image), one per destination buffer: a frame is ~40
  // launches and the host needs ~1.1 ms to enqueue them one by one (measured, bench e2e), about the GPU time itself
  struct GraphEntry { float *out3; cudaGraphExec_t exec; uint64_t launches, last_use; };
  std::vector<GraphEntry> graphs;
  uint64_t use_clock = 0;
  int eager_runs = 0;
  ~Plan() {
    for (GraphEntry &g : graphs) cudaGraphExecDestroy(g.exec);
    for (void *p : allocs) cudaFree(p);
  }
};

}  // namespace fav

using namespace fav;

struct fav_net {
  std::string arch;
  std::string padding_type = "reflect-start";
  float tanh_c = 150.f;
  int in_dim = 7;
  int reflect_pad = 0;
  bool bn = false;  // use_instance_norm = 0: SpatialBatchNormalization in evaluate mode (models_video.lua:21-25,33-37,121-127)
  std::vector<Param> params;
  std::vector<ConvDef> convs;
  std::vector<InDef> inorms;
  std::vector<SpecOp> ops;
  bool finalized = false;
  int conv_impl = 0;
  int single = 0;  // fav_net_set_precision: 1 = "fp16", one MMA per K step (ConvJob::single); 0 = "pair"
  int num_sms = 148;
  cudaStream_t cap_stream = nullptr;  // graph capture happens here (the caller's stream may be the legacy default stream)
  int device = 0;
  std::map<std::tuple<int, int, int>, std::unique_ptr<Plan>> plans;  // (B, H, W)
  Plan *last_plan = nullptr;
  size_t budget = kMaxPlanBytes;  // activation bytes of plans created from now on (fav_net_set_activation_budget)
  // style bank (fav_net_add_style): every parameter buffer holds nstyles copies, bank[buffer] bytes apart (style 0: the net's
  // own parameters); d_unscale[conv]: 2^-w_exp of each style (kMaxBatch floats, allocated by the first add_style).
  // batch_styles: the style of each image of later calls (fav_net_set_batch_styles), empty = style 0 for every image
  int nstyles = 1;
  std::map<const void *, size_t> bank;
  std::vector<float *> d_unscale;
  std::vector<int> batch_styles;
  std::vector<void *> allocs;
  ~fav_net() {
    plans.clear();
    if (cap_stream) cudaStreamDestroy(cap_stream);
    for (void *p : allocs) cudaFree(p);
  }
};

namespace fav {

static int add_param(fav_net *net, const std::string &name, std::initializer_list<int64_t> shape) {
  Param p;
  p.name = name;
  int i = 0;
  p.numel = 1;
  for (int64_t s : shape) {
    p.shape[i++] = s;
    p.numel *= s;
  }
  net->params.push_back(std::move(p));
  return (int)net->params.size() - 1;
}

static int add_conv(fav_net *net, const std::string &name, int cin, int cout, int k, int stride, int pad, bool tr,
                    int adj) {
  ConvDef c;
  init_conv_def(c, name, cin, cout, k, stride, pad, tr, adj);
  build_phases(c);
  if (tr) c.pw = add_param(net, name + ".weight", {cin, cout, k, k});
  else c.pw = add_param(net, name + ".weight", {cout, cin, k, k});
  c.pb = add_param(net, name + ".bias", {cout});
  net->convs.push_back(std::move(c));
  return (int)net->convs.size() - 1;
}
static int add_in(fav_net *net, const std::string &name, int C, int conv) {
  InDef n;
  n.name = name; n.C = C;
  n.pw = add_param(net, name + ".weight", {C});
  n.pb = add_param(net, name + ".bias", {C});
  if (net->bn) {
    n.pm = add_param(net, name + ".running_mean", {C});
    n.pv = add_param(net, name + ".running_var", {C});
    n.pe = add_param(net, name + ".eps", {1});
    n.conv = conv;
  }
  net->inorms.push_back(std::move(n));
  return (int)net->inorms.size() - 1;
}

// a parameter buffer of one style: its size rounded up to 256 bytes is the stride of its style bank (fav_net_add_style)
template <class T>
static int dev_upload(fav_net *net, const std::vector<T> &h, T **out) {
  void *d = nullptr;
  const size_t bytes = (std::max<size_t>(h.size() * sizeof(T), 16) + 255) / 256 * 256;
  FAV_TRY(check_cuda(cudaMalloc(&d, bytes), "cudaMalloc(weights)"));
  net->allocs.push_back(d);
  net->bank[d] = bytes;
  FAV_TRY(check_cuda(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice), "cudaMemcpy(weights)"));
  *out = (T *)d;
  return FAV_OK;
}

// packed tensor-core weights of every phase of c (K-step tables from plan_conv_nblocks)
static int pack_tc_weights(fav_net *net, ConvDef &c, const std::vector<float> &w) {
  for (auto &ph : c.phases) {
    std::vector<uint16_t> pk = pack_phase_weights(c, ph, w);
    uint16_t *d = nullptr;
    FAV_TRY(dev_upload(net, pk, &d));
    ph.d_b_tc = reinterpret_cast<uint4 *>(d);
  }
  return FAV_OK;
}

// w: the weights the tensor cores multiply with, b the bias; w_simt: the CUDA-core comparator's weights; scale: empty, or the
// per-channel BatchNorm scale the operand epilogue applies (fold_batch_norms).  The tensor cores get w times 2^c.w_exp
// (set_weight_prescale); the operand epilogue takes the 2^-w_exp back with the scale, every other epilogue from ConvJob::w_unscale.
static int pack_conv_weights(fav_net *net, ConvDef &c, const std::vector<float> &w, const std::vector<float> &b,
                             const std::vector<float> &w_simt, const std::vector<float> &scale) {
  set_weight_prescale(c, w);
  std::vector<float> bias(c.Npad, 0.f), sc(c.Npad, 0.f);
  for (int i = 0; i < c.cout; ++i) bias[i] = b[i];
  for (size_t i = 0; i < scale.size(); ++i) sc[i] = ldexpf(scale[i], -c.w_exp);
  FAV_TRY(dev_upload(net, bias, &c.d_bias));
  if (!scale.empty()) FAV_TRY(dev_upload(net, sc, &c.d_scale));
  for (size_t b = 0; b < c.nblock.size(); ++b) {  // N blocks: weight, bias and scale slices
    ConvDef &cb = c.nblock[b];
    std::vector<float> bb(cb.Npad, 0.f), sb(cb.Npad, 0.f);
    for (int i = 0; i < cb.cout; ++i) { bb[i] = bias[b * kMaxNBlock + i]; sb[i] = sc[b * kMaxNBlock + i]; }
    FAV_TRY(dev_upload(net, bb, &cb.d_bias));
    if (!scale.empty()) FAV_TRY(dev_upload(net, sb, &cb.d_scale));
    FAV_TRY(pack_tc_weights(net, cb, conv_nblock_weights(w, c.cin, c.cout, c.k, (int)b, c.transposed)));
  }
  for (auto &ph : c.phases) {
    // CUDA-core comparator layout: [tap][Cin_pad][Cout_pad8]
    std::vector<float> ws((size_t)ph.taps.size() * c.cin_pad * c.cout_pad8, 0.f);
    for (size_t t = 0; t < ph.taps.size(); ++t)
      for (int ci = 0; ci < c.cin; ++ci)
        for (int co = 0; co < c.cout; ++co)
          ws[(t * c.cin_pad + ci) * c.cout_pad8 + co] = weight_at(c, w_simt, co, ci, ph.taps[t].ky, ph.taps[t].kx);
    FAV_TRY(dev_upload(net, ws, &ph.d_w_simt));
  }
  if (c.nblock.empty()) FAV_TRY(pack_tc_weights(net, c, w));
  if (!c.stack.empty()) {  // stacked sub-pixel phases: column s * Cout + co holds channel co of phase s
    FAV_TRY(dev_upload(net, stack_bias(c, b), &c.d_stack_bias));
    for (ConvPhase &ph : c.stack) {
      uint16_t *d = nullptr;
      FAV_TRY(dev_upload(net, pack_phase_weights(c, ph, w), &d));
      ph.d_b_tc = reinterpret_cast<uint4 *>(d);
    }
  }
  if (c.has_fold) {  // transposed conv: one tcgen05 job for all four sub-pixel phases
    std::vector<uint16_t> pk = pack_phase_fold(c, c.fold, w);
    uint16_t *d = nullptr;
    FAV_TRY(dev_upload(net, pk, &d));
    c.fold.d_b_tc = reinterpret_cast<uint4 *>(d);
  }
  return FAV_OK;
}

// The bias each convolution runs with, its folded weights and its per-channel scale.  A batch-normalized net folds every
// inference-mode BatchNorm that directly follows a convolution into it, in double: s = weight / sqrt(running_var + eps),
// W' = W s along the output channel (dimension 1 of a transposed conv's [Cin][Cout][k][k]), b' = (b - running_mean) s + bias.
// The CUDA-core comparator multiplies with W' (fp32).  The tensor cores keep W and the operand epilogue computes acc s + b':
// W' is often tiny (s ~ 1e-2 after a first conv whose input is in pixel units), and the lo half of its fp16 hi/lo split then
// falls into the fp16 subnormals (DESIGN.md 4.1: folded weights put the net-space output 0.033 off the fp64 oracle).
// The BN of a UX token comes after the upsampling, behind the previous layer's ReLU, so it is kept as the affine
// (x - running_mean) s + bias (h_mean / h_scale).
static int fold_batch_norms(fav_net *net, std::vector<std::vector<float>> &w, std::vector<std::vector<float>> &b,
                            std::vector<std::vector<float>> &scale) {
  w.resize(net->convs.size()); b.resize(net->convs.size()); scale.assign(net->convs.size(), {});
  for (size_t i = 0; i < net->convs.size(); ++i) { w[i] = net->params[net->convs[i].pw].host; b[i] = net->params[net->convs[i].pb].host; }
  if (!net->bn) return FAV_OK;
  for (InDef &n : net->inorms) {
    const std::vector<float> &g = net->params[n.pw].host, &be = net->params[n.pb].host, &m = net->params[n.pm].host,
                             &v = net->params[n.pv].host;
    const double eps = net->params[n.pe].host[0];
    std::vector<double> sc(n.C);
    for (int ch = 0; ch < n.C; ++ch) {
      const double d = (double)v[ch] + eps;
      if (!std::isfinite(d) || !(d > 0) || !std::isfinite(g[ch]) || !std::isfinite(be[ch]) || !std::isfinite(m[ch])) {
        set_error("batch norm %s, channel %d: weight %g, bias %g, running_mean %g, running_var + eps %g (all must be finite, "
                  "running_var + eps > 0)", n.name.c_str(), ch, g[ch], be[ch], m[ch], d);
        return FAV_ERR_INVALID;
      }
      sc[ch] = (double)g[ch] / std::sqrt(d);
    }
    if (n.conv < 0) {
      n.h_mean = m;
      n.h_scale.resize(n.C);
      for (int ch = 0; ch < n.C; ++ch) n.h_scale[ch] = (float)sc[ch];
      continue;
    }
    const ConvDef &c = net->convs[n.conv];
    const int64_t kk = (int64_t)c.k * c.k;
    std::vector<float> &wc = w[n.conv], &bc = b[n.conv];
    for (int64_t i = 0; i < (int64_t)wc.size(); ++i) {
      const int co = (int)(c.transposed ? (i / kk) % c.cout : i / (kk * c.cin));
      wc[i] = (float)((double)wc[i] * sc[co]);
    }
    for (int co = 0; co < c.cout; ++co) bc[co] = (float)(((double)bc[co] - m[co]) * sc[co] + be[co]);
    scale[n.conv].assign(sc.begin(), sc.end());
  }
  return FAV_OK;
}

// ---- plan ---------------------------------------------------------------------------------------------------
static int alloc_zero(Plan &pl, void **out, size_t bytes) {
  pl.bytes += bytes;
  if (pl.dry) { *out = nullptr; return FAV_OK; }
  if (pl.bytes > pl.budget) {
    set_error("a batch of %d frames of %dx%d needs more than %.2f GiB of activations (the activation budget, "
              "fav_net_set_activation_budget): use a smaller batch", pl.B, pl.W, pl.H, pl.budget / 1073741824.0);
    return FAV_ERR_INVALID;
  }
  FAV_TRY(check_cuda(cudaMalloc(out, bytes), "cudaMalloc(activations)"));
  pl.allocs.push_back(*out);
  return check_cuda(cudaMemset(*out, 0, bytes), "cudaMemset(activations)");
}

// operand feeding convolution `c` (its pad / parity requirements)
static int make_operand(Plan &pl, int C, int H, int W, const ConvDef *consumer, int *index) {
  Operand o = operand_geometry(C, H, W, consumer);
  o.img16 = (int64_t)o.elems16;
  const size_t i = pl.ops.size();
  if (i < pl.preset.size() && pl.preset[i].first) {
    o.hi = pl.preset[i].first; o.lo = pl.preset[i].second;
  } else {
    FAV_TRY(alloc_zero(pl, (void **)&o.hi, pl.B * o.elems16 * 16));
    FAV_TRY(alloc_zero(pl, (void **)&o.lo, pl.B * o.elems16 * 16));
  }
  pl.ops.push_back(o);
  *index = (int)pl.ops.size() - 1;
  return FAV_OK;
}

// a job of conv `conv` in a plan with a style table: image b runs the weights, bias, epilogue scale and 2^-w_exp of style
// pl.styles[b] (style_at, conv.cuh).  The bias and the epilogue scale are both Npad floats, so one stride serves both.
static void set_job_styles(const fav_net *net, const Plan &pl, ConvJob &j, int conv) {
  if (!pl.styles) return;
  j.img_style = pl.styles;
  j.w_unscale_style = net->d_unscale[conv];
  j.b_style16 = (int64_t)(net->bank.at(j.b) / 16);
  j.bias_style = (int)(net->bank.at(j.bias) / 4);
}

// tensor-core jobs of c (one per phase, per N block when Cout > kMaxNBlock, or the stacked-phase jobs of plan_phase_stack) and
// CUDA-core comparator jobs (one per phase); stats: the [sum][sum of squares] slots of c's output for the fused InstanceNorm
// statistics, or null; epi (batch-normalized nets): the operand step whose ReLU / skip / packing the tensor-core epilogue
// performs (set_opnd_epilogue), or null.  FAV_NO_STACK keeps one job per phase, so one process can compare the two plans.
static int build_conv_jobs(fav_net *net, Plan &pl, PlanStep &st, const ConvDef &c, bool last, float *out3, double *stats,
                           const PlanStep *epi = nullptr) {
  const Operand &in = pl.ops[st.src];
  const int nb = c.nblock.empty() ? 1 : (int)c.nblock.size();
  const bool stack = !c.stack.empty() && !epi && !getenv("FAV_NO_STACK");
  for (int b = 0; b < nb; ++b) {
    const ConvDef &cd = c.nblock.empty() ? c : c.nblock[b];
    float *raw = st.raw.p + conv_nblock_raw_offset(b, st.raw.Wp);
    bool fold_done = false;
    for (const ConvPhase &ph : stack ? c.stack : cd.phases) {
      const bool use_fold = cd.has_fold && !getenv("FAV_NO_FOLD");
      ConvJob j;
      if (use_fold) {
        if (!fold_done) {
          FAV_TRY(fill_conv_job(cd, cd.fold, in, j));
          set_conv_batch(j, pl.B, st.raw.img, 3ll * pl.H * pl.W, pl.stats_img);
          j.b = cd.fold.d_b_tc; j.bias = cd.d_bias;
          j.raw = raw; j.raw_Cq = st.raw.Cq; j.raw_Wp = st.raw.Wp;
          j.final_mode = 0; j.out3 = out3; j.tanh_c = net->tanh_c;
          conv_nblock_stats(j, stats, c.cout, b);
          j.single = net->single;
          set_job_styles(net, pl, j, (int)(&c - net->convs.data()));
          conv_tc_choose_slots(j);
          if (const char *e = getenv("FAV_DBG")) j.dbg = atoi(e);
          if (conv_tc_smem_bytes(j) > 227 * 1024) { set_error("conv %s: shared memory budget exceeded (fold)", c.name.c_str()); return FAV_ERR_UNSUPPORTED; }
          st.tc.push_back(j);
          fold_done = true;
        }
      } else {
        FAV_TRY(fill_conv_job(cd, ph, in, j));
        set_conv_batch(j, pl.B, st.raw.img, 3ll * pl.H * pl.W, pl.stats_img);
        j.b = ph.d_b_tc; j.bias = stack ? c.d_stack_bias : cd.d_bias;
        j.raw = raw; j.raw_Cq = st.raw.Cq; j.raw_Wp = st.raw.Wp;
        j.final_mode = last ? 1 : 0; j.out3 = out3; j.tanh_c = net->tanh_c;
        conv_nblock_stats(j, stats, c.cout, b);
        if (epi)
          set_opnd_epilogue(j, b, cd.d_scale, pl.ops[epi->dst], epi->relu, epi->skip >= 0 ? &pl.ops[epi->skip] : nullptr, epi->shave);
        j.single = net->single;  // the norm-on-load copies (fuse_norm_on_load) and tc_plain keep it
        set_job_styles(net, pl, j, (int)(&c - net->convs.data()));
        conv_tc_choose_slots(j);
        if (const char *e = getenv("FAV_DBG")) j.dbg = atoi(e);
        if (conv_tc_smem_bytes(j) > 227 * 1024) {
          set_error("conv %s: shared memory budget exceeded", c.name.c_str());
          return FAV_ERR_UNSUPPORTED;
        }
        st.tc.push_back(j);
      }
    }
  }
  for (const ConvPhase &ph : c.phases) {
    SimtJob s;
    memset(&s, 0, sizeof(s));
    s.in = in; s.sy = s.sx = c.in_stride; s.ntaps = (int)ph.taps.size();
    for (int t = 0; t < s.ntaps; ++t) { s.tdy[t] = (int8_t)ph.taps[t].dy; s.tdx[t] = (int8_t)ph.taps[t].dx; }
    s.w = ph.d_w_simt; s.Cin_pad = c.cin_pad; s.Cout = c.cout; s.Cout_pad8 = c.cout_pad8; s.bias = c.d_bias;
    s.Ho = c.transposed ? in.H : st.raw.H; s.Wo = c.transposed ? in.W : st.raw.W; s.raw = st.raw.p; s.raw_Cq = st.raw.Cq; s.raw_Wp = st.raw.Wp;
    s.raw_planar = st.raw.planar; s.raw_Hp = st.raw.Hp;
    s.oy_mul = s.ox_mul = c.out_mul; s.oy_off = ph.oy_off; s.ox_off = ph.ox_off;
    s.final_mode = last ? 1 : 0; s.out3 = out3; s.tanh_c = net->tanh_c;
    st.simt.push_back(s);
  }
  return FAV_OK;
}

// Fold the InstanceNorm (+ReLU) pass just planned (the last step) into the patch producers of conv step cs, its only reader:
// the pass then never runs and cs normalises the raw tensor while it loads it (conv_tc.cu norm-on-load).  Not for a pass that
// adds a skip or whose operand a later step reads as a skip (src_is_skip: the first conv of a residual block), and only when
// every job of cs has a patch layout the producers can fill (nl_geometry_ok) and still fits shared memory.  Each N block of a
// wide conv normalises the whole patch itself; the per-channel tables hold at most 256 channels (conv_tc.cu kNlMaxC).  The
// unfused jobs stay in cs.tc_plain for fav_net_layer_output (run_plan's replay).  FAV_NO_NL switches every fusion off.
// The x-fold final conv stays unfused although the producers could fill its patch: it normalises every raw pixel once per
// filter row and ran slower fused than the pass it would remove (DESIGN.md 4.1, H100 at 720p: 0.485 ms against 0.271 ms
// + a 0.086 ms pass).
static void fuse_norm_on_load(fav_net *net, Plan &pl, PlanStep &cs, bool src_is_skip) {
  if (net->bn || src_is_skip || pl.steps.empty() || getenv("FAV_NO_NL")) return;
  PlanStep &ap = pl.steps.back();
  if (ap.kind != 1 || ap.skip >= 0 || ap.dst != cs.src) return;
  const InDef &n = net->inorms[ap.inorm];
  if (n.C > 256) return;
  std::vector<ConvJob> fused;
  for (const ConvJob &j : cs.tc) {
    if (!nl_geometry_ok(j) || j.xfold_kw) return;
    ConvJob t = j;
    set_norm_on_load(t, ap.raw, pl.ops[cs.src], ap.relu, pl.stats + ap.stats_off, pl.stats_img, n.d_gamma, n.d_beta);
    if (t.img_style) t.nl_style = (int)(net->bank.at(n.d_gamma) / 4);
    conv_tc_choose_slots(t);
    if (conv_tc_smem_bytes(t) > 227 * 1024 || !(t.b_resident || t.b_slots >= 2)) return;
    fused.push_back(t);
  }
  if (fused.empty()) return;
  cs.tc_plain = std::move(cs.tc);
  cs.tc = std::move(fused);
  ap.fused_nl = true;
}

// the buffers and steps of plan pl (B, H, W, budget, dry and preset set by the caller)
static int build_plan_steps(fav_net *net, Plan *pl) {
  const int B = pl->B, H = pl->H, W = pl->W;
  const int R = net->reflect_pad;
  if (R >= H || R >= W) { set_error("frame smaller than the reflection padding (%d)", R); return FAV_ERR_INVALID; }
  // pass 1: sizes -> largest raw tensor, stats slots
  size_t raw_max = 0;
  int stats_slots = 0;
  {
    int h = H + 2 * R, w = W + 2 * R;
    for (auto &op : net->ops) {
      if (op.kind == 2) { h *= op.scale; w *= op.scale; stats_slots += net->bn ? 0 : 2 * net->inorms[op.inorm[0]].C; continue; }
      int n = op.kind == 1 ? 2 : 1;
      for (int i = 0; i < n; ++i) {
        const ConvDef &c = net->convs[op.conv[i]];
        int ho, wo;
        conv_out_size(c, h, w, &ho, &wo);
        raw_max = std::max(raw_max, (size_t)(ho + 2) * round_up(c.cout, 4) * round_up(wo, kTileM));
        h = ho; w = wo;
        if (op.inorm[i] >= 0 && !net->bn) stats_slots += 2 * c.cout;
      }
    }
    // the final conv writes a [3][H][W] frame per image: a net that returns another size would write past it (and into the
    // next image of a batch).  Every stride-2 layer needs an even input to be undone exactly by the upsampling layers.
    if (h != H || w != W) {
      int n2 = 0;
      for (const ConvDef &c : net->convs) n2 += c.in_stride == 2;
      set_error("frame size %dx%d: this arch would return a %dx%d frame; with its %d stride-2 layers H and W must be "
                "multiples of %d (when its residual blocks sit at the lowest resolution)", W, H, w, h, n2, 1 << n2);
      return FAV_ERR_INVALID;
    }
  }
  pl->raw_bytes = raw_max * sizeof(float) + 4096;  // per image (a multiple of 16 bytes)
  if (!net->bn) {  // a batch-normalized net's tensor-core epilogues write operands, not raw tensors
    FAV_TRY(alloc_zero(*pl, (void **)&pl->raw_buf, B * pl->raw_bytes));
    FAV_TRY(alloc_zero(*pl, (void **)&pl->raw_buf2, B * pl->raw_bytes));
  }
  pl->stats_img = std::max(1, stats_slots);
  pl->stats_bytes = B * pl->stats_img * sizeof(double);
  FAV_TRY(alloc_zero(*pl, (void **)&pl->stats, pl->stats_bytes));
  FAV_TRY(alloc_zero(*pl, (void **)&pl->msb, std::max(1, stats_slots) * 2 * sizeof(float)));
  FAV_TRY(alloc_zero(*pl, (void **)&pl->in7, (size_t)B * net->in_dim * H * W * sizeof(float)));
  FAV_TRY(alloc_zero(*pl, (void **)&pl->out3, (size_t)B * 3 * H * W * sizeof(float)));

  // flat list of convs in execution order, to look up the consumer of each operand
  std::vector<int> order;
  for (auto &op : net->ops) {
    if (op.kind == 2) continue;
    order.push_back(op.conv[0]);
    if (op.kind == 1) order.push_back(op.conv[1]);
  }
  size_t pos = 0;
  int cur;
  FAV_TRY(make_operand(*pl, net->in_dim, H + 2 * R, W + 2 * R, &net->convs[order[0]], &cur));
  int stats_off = 0;
  for (size_t oi = 0; oi < net->ops.size(); ++oi) {
    const SpecOp &op = net->ops[oi];
    if (op.kind == 2) {  // UX: operand -> upsampled, normalised operand for the next convolution
      PlanStep us;
      us.kind = 2; us.scale = op.scale; us.inorm = op.inorm[0]; us.src = cur; us.relu = 1; us.stats_off = stats_off;
      const int C = net->inorms[op.inorm[0]].C;
      if (!net->bn) stats_off += 2 * C;
      const ConvDef *consumer = pos < order.size() ? &net->convs[order[pos]] : nullptr;
      FAV_TRY(make_operand(*pl, C, pl->ops[cur].H * op.scale, pl->ops[cur].W * op.scale, consumer, &us.dst));
      cur = us.dst;
      us.layer_index = (int)oi;
      pl->layer_operand[(int)oi] = cur;
      pl->steps.push_back(std::move(us));
      continue;
    }
    const int n = op.kind == 1 ? 2 : 1;
    const int block_in = cur;
    for (int i = 0; i < n; ++i, ++pos) {
      const ConvDef &c = net->convs[op.conv[i]];
      PlanStep cs;
      cs.kind = 0; cs.conv = op.conv[i]; cs.src = cur;
      int ho, wo;
      conv_out_size(c, pl->ops[cur].H, pl->ops[cur].W, &ho, &wo);
      cs.raw.p = (pos & 1) ? pl->raw_buf2 : pl->raw_buf; cs.raw_sel = (int)(pos & 1);
      cs.raw.C = c.cout; cs.raw.Cq = round_up(c.cout, 4) / 4; cs.raw.H = ho; cs.raw.W = wo;
      cs.raw.Hp = ho + 2; cs.raw.Wp = round_up(wo, kTileM); cs.raw.img = (int64_t)(pl->raw_bytes / sizeof(float));
      const bool last = op.last && i == n - 1;
      if (last) {
        FAV_TRY(build_conv_jobs(net, *pl, cs, c, true, nullptr, nullptr));
        fuse_norm_on_load(net, *pl, cs, false);
        cs.layer_index = (int)oi;
        pl->steps.push_back(std::move(cs));
        break;
      }
      // InstanceNorm / BatchNorm (+ReLU) (+skip) -> operand for the next convolution
      if (op.inorm[i] < 0 || c.cout % 8) {
        set_error("layer %s: a non-final convolution must be followed by InstanceNormalization (Cout %% 8 == 0)",
                  c.name.c_str());
        return FAV_ERR_UNSUPPORTED;
      }
      PlanStep ns;
      ns.kind = 1; ns.inorm = op.inorm[i]; ns.raw = cs.raw; ns.raw_sel = cs.raw_sel; ns.stats_off = stats_off;
      if (!net->bn) stats_off += 2 * c.cout;
      const ConvDef *consumer = pos + 1 < order.size() ? &net->convs[order[pos + 1]] : nullptr;
      FAV_TRY(make_operand(*pl, c.cout, ho, wo, consumer, &ns.dst));
      if (op.kind == 1) {
        ns.relu = i == 0 ? 1 : (op.relu ? 1 : 0);               // CX: needs_relu after the block (models_video.lua:108)
        ns.skip = (i == 1 && op.skip) ? block_in : -1;          // RX: ShaveImage(2) / Identity of the block input (:46-50)
        ns.shave = op.shave;
      } else {
        ns.relu = op.relu ? 1 : 0;
      }
      // InstanceNorm: statistics fused into the epilogue.  BatchNorm (folded into the conv): the epilogue performs ns itself,
      // which then only runs after the CUDA-core comparator
      FAV_TRY(build_conv_jobs(net, *pl, cs, c, false, nullptr, net->bn ? nullptr : pl->stats + ns.stats_off,
                              net->bn ? &ns : nullptr));
      fuse_norm_on_load(net, *pl, cs, op.kind == 1 && i == 0 && op.skip);
      pl->steps.push_back(std::move(cs));
      cur = ns.dst;
      if (i == n - 1) { ns.layer_index = (int)oi; pl->layer_operand[(int)oi] = cur; }
      pl->steps.push_back(std::move(ns));
    }
  }
  return FAV_OK;
}

// the plan's steps as the buffer planner sees them.  A batch-normalized net's conv epilogue writes the next operand (and reads
// the skip) itself; the norm step after it does the same on the CUDA-core comparator.
static std::vector<ArenaStep> arena_steps(const fav_net *net, const Plan &pl) {
  std::vector<ArenaStep> v(pl.steps.size());
  for (size_t si = 0; si < pl.steps.size(); ++si) {
    const PlanStep &s = pl.steps[si];
    ArenaStep &a = v[si];
    if (s.kind != 1) a.src = s.src;
    if (s.kind != 0) { a.dst = s.dst; a.skip = s.skip; }
    if (s.kind == 0 && net->bn && si + 1 < pl.steps.size() && pl.steps[si + 1].kind == 1) {
      a.dst = pl.steps[si + 1].dst; a.skip = pl.steps[si + 1].skip;
    }
  }
  return v;
}

// The activation bytes of a (B, H, W) plan with every operand in its own buffer (all_live) and with the operands in one arena
// (arena_plan.hpp; *ap, when given, receives the arena layout).  The network's first operand stays out of the arena: the
// temporal-stage kernels write it before the frame's steps run, and fav_net_layer_output's replay starts from it.
static int plan_sizes(fav_net *net, int B, int H, int W, size_t *all_live, size_t *arena, ArenaPlan *ap = nullptr) {
  Plan dry;
  dry.B = B; dry.H = H; dry.W = W; dry.dry = true;
  FAV_TRY(build_plan_steps(net, &dry));
  std::vector<size_t> bytes(dry.ops.size());
  std::vector<char> pinned(dry.ops.size(), 0);
  size_t own = 0;  // what the arena operands take in buffers of their own
  for (size_t i = 0; i < dry.ops.size(); ++i) {
    const size_t half = (size_t)B * dry.ops[i].elems16 * 16;  // hi, then lo at the next kArenaAlign boundary
    bytes[i] = 2 * ((half + kArenaAlign - 1) / kArenaAlign * kArenaAlign);
    if (i) own += 2 * half;
  }
  pinned[0] = 1;
  ArenaPlan p = plan_arena(arena_steps(net, dry), bytes, pinned);
  *all_live = dry.bytes;
  *arena = dry.bytes - own + p.arena_bytes;
  if (ap) *ap = std::move(p);
  return FAV_OK;
}

// A plan whose buffers fit the net's activation budget each get their own (zeroed once).  Otherwise the operands share one
// arena by lifetime; each step that writes an operand first zeroes its border (launch_clear_border).  The choice depends on
// (B, H, W) and the budget only.
static int build_plan(fav_net *net, int B, int H, int W, Plan **out) {
  if (B < 1 || B > kMaxBatch) {
    set_error("batch of %d frames: 1 to %d frames per call", B, kMaxBatch);
    return FAV_ERR_INVALID;
  }
  auto key = std::make_tuple(B, H, W);
  auto it = net->plans.find(key);
  if (it != net->plans.end()) { *out = it->second.get(); net->last_plan = *out; return FAV_OK; }
  if (H % 4 || W % 4 || H < 16 || W < 16) {
    set_error("frame size %dx%d: H and W must be multiples of 4 and at least 16 (the default arch's two stride-2 layers "
              "restore the input size only then, SURVEY appendix B)", W, H);
    return FAV_ERR_INVALID;
  }
  size_t all_live = 0, shared = 0;
  ArenaPlan ap;
  FAV_TRY(plan_sizes(net, B, H, W, &all_live, &shared, &ap));
  std::unique_ptr<Plan> pl(new Plan());
  pl->B = B; pl->H = H; pl->W = W; pl->budget = net->budget;
  if (all_live > net->budget) {
    if (shared > net->budget) {
      set_error("a batch of %d frames of %dx%d needs %.2f GiB of activations, %.2f GiB with buffers shared between layers; the "
                "activation budget is %.2f GiB (fav_net_set_activation_budget): use a smaller batch", B, W, H,
                all_live / 1073741824.0, shared / 1073741824.0, net->budget / 1073741824.0);
      return FAV_ERR_INVALID;
    }
    FAV_TRY(check_cuda(cudaMalloc(&pl->arena, ap.arena_bytes), "cudaMalloc(activation arena)"));
    pl->allocs.push_back(pl->arena);
    pl->bytes += ap.arena_bytes;
    // no operand may rely on what the arena held before its producer ran: fill it with fp16 NaNs, not zeros
    FAV_TRY(check_cuda(cudaMemset(pl->arena, 0xff, ap.arena_bytes), "cudaMemset(activation arena)"));
    pl->preset.assign(ap.off.size(), {nullptr, nullptr});
    for (size_t i = 0; i < ap.off.size(); ++i) {
      if (ap.first[i] < 0) continue;
      char *hi = (char *)pl->arena + ap.off[i];
      pl->preset[i] = {(__half *)hi, (__half *)(hi + ap.bytes[i] / 2)};  // hi, then lo
    }
    pl->kept = ap.kept;
  }
  if (net->nstyles > 1) {
    FAV_TRY(check_cuda(cudaMalloc(&pl->styles, kMaxBatch * sizeof(int)), "cudaMalloc(style table)"));
    pl->allocs.push_back(pl->styles);
    FAV_TRY(check_cuda(cudaMemset(pl->styles, 0, kMaxBatch * sizeof(int)), "cudaMemset(style table)"));
    pl->styles_host.assign(B, 0);
  }
  FAV_TRY(build_plan_steps(net, pl.get()));
  if (pl->arena) {
    for (size_t i = 0; i < pl->ops.size(); ++i) {
      if (ap.first[i] < 0) continue;
      if (pl->steps[ap.first[i]].clear >= 0) { set_error("internal: two operands become live at step %d", ap.first[i]); return FAV_ERR_INVALID; }
      pl->steps[ap.first[i]].clear = (int)i;
    }
  }
  *out = pl.get();
  net->last_plan = pl.get();
  net->plans[key] = std::move(pl);
  return FAV_OK;
}

// The plan of a call on B frames of H x W, with its style table holding the net's batch assignment (fav_net_set_batch_styles),
// written on the call's stream when it changed: the plan and its CUDA graphs stay as they are.
static int plan_for_call(fav_net *net, int B, int H, int W, cudaStream_t st, Plan **out) {
  const std::vector<int> &a = net->batch_styles;
  FAV_REQUIRE(a.empty() || (int)a.size() == B, "a call on %d frames with a style assignment for %d (fav_net_set_batch_styles): the "
              "batch must have one frame per entry, or the assignment must be cleared (n = 0)", B, (int)a.size());
  FAV_TRY(build_plan(net, B, H, W, out));
  Plan &pl = **out;
  if (!pl.styles) return FAV_OK;
  const std::vector<int> want = a.empty() ? std::vector<int>(B, 0) : a;
  if (want == pl.styles_host) return FAV_OK;
  // pageable source: staged before the call returns, ordered on st before the frame's kernels
  FAV_TRY(check_cuda(cudaMemcpyAsync(pl.styles, want.data(), B * sizeof(int), cudaMemcpyHostToDevice, st), "cudaMemcpyAsync(styles)"));
  pl.styles_host = want;
  return FAV_OK;
}

struct ProfRec {
  int kind;  // 0 pack, 1 conv, 2 in_stats(+finalize), 3 in_apply
  float ms;
  double work;  // conv: algorithmic FLOPs (logical channels); others: algorithmic bytes
  char name[24];
  cudaEvent_t e0, e1;
};

// the raw tensors of a batch-normalized net, which only the CUDA-core comparator writes: allocated at its first run
static int ensure_raw(Plan &pl) {
  if (pl.raw_buf) return FAV_OK;
  FAV_TRY(alloc_zero(pl, (void **)&pl.raw_buf, pl.B * pl.raw_bytes));
  FAV_TRY(alloc_zero(pl, (void **)&pl.raw_buf2, pl.B * pl.raw_bytes));
  for (PlanStep &s : pl.steps) {
    float *p = s.raw_sel ? pl.raw_buf2 : pl.raw_buf;
    s.raw.p = p;
    for (SimtJob &j : s.simt) j.raw = p;
  }
  return FAV_OK;
}

// in7 == nullptr: the caller has already written the first operand (fused temporal input, run_plan_frame)
// last >= 0: steps 0..last only.  unfused: the passes the plan folds into their consumers run, and the consumers read their
// operands (replay_unfused)
static int run_plan(fav_net *net, Plan &pl, const float *in7, float *out3, int final_mode, cudaStream_t st,
                    std::vector<ProfRec> *prof = nullptr, int last = -1, bool unfused = false) {
  auto begin = [&](int kind, double work, const std::string &name) -> int {
    if (!prof) return FAV_OK;
    ProfRec r;
    r.kind = kind; r.ms = 0; r.work = work;
    snprintf(r.name, sizeof(r.name), "%s", name.c_str());
    FAV_TRY(check_cuda(cudaEventCreate(&r.e0), "cudaEventCreate"));
    FAV_TRY(check_cuda(cudaEventCreate(&r.e1), "cudaEventCreate"));
    FAV_TRY(check_cuda(cudaEventRecord(r.e0, st), "cudaEventRecord"));
    prof->push_back(r);
    return FAV_OK;
  };
  auto end = [&]() -> int {
    if (!prof) return FAV_OK;
    return check_cuda(cudaEventRecord(prof->back().e1, st), "cudaEventRecord");
  };
  if (net->bn && net->conv_impl != 0) FAV_TRY(ensure_raw(pl));
  if (!net->bn) FAV_TRY(check_cuda(cudaMemsetAsync(pl.stats, 0, pl.stats_bytes, st), "cudaMemsetAsync(stats)"));
  if (in7) {
    FAV_TRY(begin(0, (double)pl.ops[0].H * pl.ops[0].W * (4.0 * net->in_dim + 32.0), "pack_input"));
    FAV_TRY(launch_pack_input(in7, net->in_dim, pl.H, pl.W, net->reflect_pad, pl.ops[0], st, pl.B));
    FAV_TRY(end());
  }
  for (size_t si = 0; si < pl.steps.size() && (last < 0 || (int)si <= last); ++si) {
    PlanStep &s = pl.steps[si];
    if (s.clear >= 0) FAV_TRY(launch_clear_border(pl.ops[s.clear], pl.B, st));
    if (s.kind == 0) {
      {
        const ConvDef &c = net->convs[s.conv];
        const Operand &in = pl.ops[s.src];
        double px = c.transposed ? (double)in.H * in.W : (double)s.raw.H * s.raw.W;
        FAV_TRY(begin(1, 2.0 * c.cin * c.cout * c.k * c.k * px, c.name));
      }
      if (net->conv_impl == 0) {
        for (ConvJob &j : (unfused && !s.tc_plain.empty()) ? s.tc_plain : s.tc) {
          if (j.final_mode) { j.final_mode = final_mode; j.out3 = out3; }
          FAV_TRY(launch_conv_tc(j, net->num_sms, st));
        }
      } else {
        for (SimtJob &j : s.simt) {
          if (j.final_mode) { j.final_mode = final_mode; j.out3 = out3; }
          for (int b = 0; b < pl.B; ++b) {  // the comparator runs one image at a time, with its style's weights and bias
            SimtJob jb = j;
            if (pl.styles) {
              const int sb = pl.styles_host[b];
              jb.w += sb * (int64_t)(net->bank.at(j.w) / 4);
              jb.bias += sb * (int64_t)(net->bank.at(j.bias) / 4);
            }
            jb.in = image_of(j.in, b);
            jb.raw = j.raw ? j.raw + b * s.raw.img : nullptr;
            jb.out3 = j.out3 ? j.out3 + (int64_t)b * 3 * pl.H * pl.W : nullptr;
            FAV_TRY(launch_conv_simt(jb, st));
          }
        }
      }
      FAV_TRY(end());
    } else if (s.kind == 2) {
      const InDef &n = net->inorms[s.inorm];
      const Operand &src = pl.ops[s.src];
      FAV_TRY(begin(3, 12.0 * n.C * src.H * src.W * (1.0 + s.scale * s.scale) / 2.0, n.name + ".up"));
      FAV_TRY(launch_up_in(src, pl.stats + s.stats_off, n.d_gamma, n.d_beta, 1e-5f, s.relu, s.scale, pl.ops[s.dst], st, n.d_mean,
                           n.d_scale, pl.B, pl.stats_img, pl.styles, pl.styles ? (int64_t)(net->bank.at(n.d_beta) / 4) : 0));
      FAV_TRY(end());
    } else {
      if (s.fused_nl && net->conv_impl == 0 && !unfused) continue;  // the consumer conv normalises while it loads (norm-on-load)
      const InDef &n = net->inorms[s.inorm];
      if (net->bn) {  // BatchNorm folded into the conv: its tensor-core epilogue wrote the operand
        if (net->conv_impl == 0) continue;
        FAV_TRY(begin(3, (s.skip >= 0 ? 12.0 : 8.0) * n.C * s.raw.H * s.raw.W, n.name + ".apply"));
        FAV_TRY(launch_in_apply(s.raw, nullptr, nullptr, nullptr, 0.f, s.relu, s.skip >= 0 ? &pl.ops[s.skip] : nullptr, s.shave,
                                pl.ops[s.dst], st, pl.B));
        FAV_TRY(end());
        continue;
      }
      double *sums = pl.stats + s.stats_off;
      const double elems = (double)n.C * s.raw.H * s.raw.W;
      if (net->conv_impl != 0) {  // the tcgen05 epilogue already accumulated the statistics
        FAV_TRY(begin(2, 4.0 * elems, n.name + ".stats"));
        FAV_TRY(launch_in_stats(s.raw, sums, st, pl.B, pl.stats_img));
        FAV_TRY(end());
      }
      // InstanceNormalization.lua:21,39: eps = 1e-5, statistics over H*W of each (n, c)
      FAV_TRY(begin(3, (s.skip >= 0 ? 12.0 : 8.0) * elems, n.name + ".apply"));
      FAV_TRY(launch_in_apply(s.raw, sums, n.d_gamma, n.d_beta, 1e-5f, s.relu, s.skip >= 0 ? &pl.ops[s.skip] : nullptr, s.shave,
                              pl.ops[s.dst], st, pl.B, pl.stats_img, pl.styles,
                              pl.styles ? (int64_t)(net->bank.at(n.d_gamma) / 4) : 0));
      FAV_TRY(end());
    }
  }
  return FAV_OK;
}

// run_[next_]image: the network part of a frame (input = pl.in7, fused deprocess) as one graph launch
static int run_plan_frame(fav_net *net, Plan &pl, const float *src7, float *out3, cudaStream_t st) {
  static const bool no_graph = getenv("FAV_NO_GRAPH") != nullptr;
  if (no_graph || net->conv_impl != 0) return run_plan(net, pl, src7, out3, 2, st);
  for (Plan::GraphEntry &g : pl.graphs)
    if (g.out3 == out3) {
      g.last_use = ++pl.use_clock;
      FAV_TRY(check_cuda(cudaGraphLaunch(g.exec, st), "cudaGraphLaunch"));
      g_launches.fetch_add(g.launches, std::memory_order_relaxed);
      return FAV_OK;
    }
  if (pl.eager_runs < 1) {  // one-time lazy initialisation (function attributes) must happen outside a capture
    ++pl.eager_runs;
    return run_plan(net, pl, src7, out3, 2, st);
  }
  if (!net->cap_stream)
    FAV_TRY(check_cuda(cudaStreamCreateWithFlags(&net->cap_stream, cudaStreamNonBlocking), "cudaStreamCreate(capture)"));
  const uint64_t l0 = g_launches.load();
  FAV_TRY(check_cuda(cudaStreamBeginCapture(net->cap_stream, cudaStreamCaptureModeRelaxed), "cudaStreamBeginCapture"));
  const int rc = run_plan(net, pl, src7, out3, 2, net->cap_stream);
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(net->cap_stream, &graph);
  const uint64_t n = g_launches.load() - l0;
  g_launches.fetch_sub(n, std::memory_order_relaxed);  // captured, not executed
  if (rc != FAV_OK || ce != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    if (rc != FAV_OK) return rc;
    return run_plan(net, pl, src7, out3, 2, st);
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) {
    cudaGetLastError();
    return run_plan(net, pl, src7, out3, 2, st);
  }
  if (pl.graphs.size() >= 8) {  // evict the least recently used destination
    size_t v = 0;
    for (size_t i = 1; i < pl.graphs.size(); ++i)
      if (pl.graphs[i].last_use < pl.graphs[v].last_use) v = i;
    cudaGraphExecDestroy(pl.graphs[v].exec);
    pl.graphs.erase(pl.graphs.begin() + v);
  }
  pl.graphs.push_back(Plan::GraphEntry{out3, exec, n, ++pl.use_clock});
  FAV_TRY(check_cuda(cudaGraphLaunch(exec, st), "cudaGraphLaunch"));
  g_launches.fetch_add(n, std::memory_order_relaxed);
  return FAV_OK;
}

}  // namespace fav

// =============================================================================================================
extern "C" {

int fav_net_create(const char *arch, const char *padding_type, float tanh_constant, int in_dim, fav_net_t **out) {
  return fav_net_create_norm(arch, padding_type, tanh_constant, in_dim, "instance", out);
}

int fav_net_create_norm(const char *arch, const char *padding_type, float tanh_constant, int in_dim, const char *norm,
                        fav_net_t **out) {
  FAV_REQUIRE(arch && out, "fav_net_create: null argument");
  // train_video.lua:22 -use_instance_norm: 1 = InstanceNormalization, 0 = SpatialBatchNormalization (models_video.lua:21-25,
  // 33-37,121-127), which get_model runs in evaluate mode (fast_artistic_video_core.lua:46)
  const std::string nt = norm ? norm : "instance";
  FAV_REQUIRE(nt == "instance" || nt == "batch", "fav_net_create_norm: norm must be 'instance' or 'batch' (got '%s')", nt.c_str());
  FAV_REQUIRE(in_dim >= 1 && in_dim <= 8, "fav_net_create: in_dim must be in [1,8] (video nets use 7, image nets 3)");
  // models_video.lua:13-19,27-31,46-50,71-79: 'reflect-start' (every released video model; train_video.lua:25) = unpadded
  // residual convs + ShaveImage(2) + one lazily inserted reflection pad (train_video.lua:319-324); 'zero' = residual convs with
  // zero padding 1 and an Identity skip.  'reflect' / 'replicate' put a padding module in front of EVERY convolution and 'none'
  // returns a smaller frame than it was given: not built (no released model uses them).
  const std::string ptype = padding_type ? padding_type : "reflect-start";
  if (ptype != "reflect-start" && ptype != "zero") {
    set_error("padding_type '%s' is not supported (supported: 'reflect-start', the released video models' setting "
              "(train_video.lua:25), and 'zero')", ptype.c_str());
    return FAV_ERR_UNSUPPORTED;
  }
  const bool zero_pad = ptype == "zero";
  std::unique_ptr<fav_net> net(new fav_net());
  net->arch = arch; net->tanh_c = tanh_constant; net->in_dim = in_dim; net->padding_type = ptype; net->bn = nt == "batch";
  // tokenise (models_video.lua:56)
  std::vector<std::string> toks;
  {
    std::string s(arch), cur;
    for (char ch : s) {
      if (ch == ',') { toks.push_back(cur); cur.clear(); }
      else if (ch != ' ') cur.push_back(ch);
    }
    if (!cur.empty()) toks.push_back(cur);
  }
  FAV_REQUIRE(!toks.empty(), "fav_net_create: empty arch");
  int prev = in_dim;
  double scale = 1.0, shrink = 0.0;
  for (size_t i = 0; i < toks.size(); ++i) {
    const std::string &v = toks[i];
    const std::string name = "l" + std::to_string(i);
    SpecOp op;
    op.kind = 0; op.relu = true; op.last = (i + 1 == toks.size());
    bool needs_bn = true;
    int next = 0;
    char c0 = v[0];
    if (c0 == 'c' && v.size() >= 6 && v[2] == 's' && v[4] == '-') {  // cXsY-Z  models_video.lua:65-80
      int f = v[1] - '0', s = v[3] - '0';
      next = atoi(v.c_str() + 5);
      FAV_REQUIRE(f % 2 == 1 && (s == 1 || s == 2) && next > 0, "bad arch token '%s'", v.c_str());
      op.conv[0] = add_conv(net.get(), name, prev, next, f, s, (f - 1) / 2, false, 0);
      if (s == 2) scale *= 2;
    } else if (c0 == 'd') {  // dX  :90-93
      next = atoi(v.c_str() + 1);
      FAV_REQUIRE(next > 0, "bad arch token '%s'", v.c_str());
      op.conv[0] = add_conv(net.get(), name, prev, next, 3, 2, 1, false, 0);
      scale *= 2;
    } else if (c0 == 'u') {  // uX  :99-102  SpatialFullConvolution(3,3,2,2,1,1,1,1)
      next = atoi(v.c_str() + 1);
      FAV_REQUIRE(next > 0, "bad arch token '%s'", v.c_str());
      op.conv[0] = add_conv(net.get(), name, prev, next, 3, 2, 1, true, 1);
      scale /= 2;
    } else if (c0 == 'U') {  // UX  :94-98  SpatialUpSamplingNearest(X), followed by IN + ReLU (:121-130)
      int sc = atoi(v.c_str() + 1);
      FAV_REQUIRE(sc >= 1 && sc <= 4 && !op.last && prev % 8 == 0, "bad arch token '%s'", v.c_str());
      next = prev;
      op.kind = 2; op.scale = sc;
      op.inorm[0] = add_in(net.get(), name + ".n", next, -1);
      needs_bn = false;
      scale /= sc;
    } else if (c0 == 'f' && v.size() >= 6 && v[2] == 's' && v[4] == '-') {  // fXsY-Z  :81-89  SpatialFullConvolution(f,f,s,s,p,p,s-1,s-1)
      int f = v[1] - '0', st = v[3] - '0';
      next = atoi(v.c_str() + 5);
      FAV_REQUIRE(f % 2 == 1 && (st == 1 || st == 2) && next > 0, "bad arch token '%s'", v.c_str());
      op.conv[0] = add_conv(net.get(), name, prev, next, f, st, (f - 1) / 2, true, st - 1);
      scale /= st;
    } else if (c0 == 'R' || c0 == 'C') {  // RX :109-114 residual block; CX :103-108 the same conv block without the skip
      next = atoi(v.c_str() + 1);
      FAV_REQUIRE(next == prev, "block %c%d needs %d input channels (got %d)", c0, next, next, prev);
      const int bp = zero_pad ? 1 : 0;  // build_conv_block :12-20
      op.kind = 1;
      op.skip = c0 == 'R';
      op.shave = zero_pad ? 0 : 2;      // ShaveImage(2) vs Identity :46-50
      op.conv[0] = add_conv(net.get(), name + ".c1", prev, next, 3, 1, bp, false, 0);
      op.inorm[0] = add_in(net.get(), name + ".n1", next, op.conv[0]);
      op.conv[1] = add_conv(net.get(), name + ".c2", next, next, 3, 1, bp, false, 0);
      op.inorm[1] = add_in(net.get(), name + ".n2", next, op.conv[1]);
      needs_bn = false; op.relu = c0 == 'C';  // :107-108, :113-114
      if (!zero_pad) shrink += 4 * scale;
    } else {
      set_error("arch token '%s' is not supported by the sm_90a path (supported: cXsY-Z, fXsY-Z, dX, uX, UX, CX, RX)", v.c_str());
      return FAV_ERR_UNSUPPORTED;
    }
    if (op.last) { needs_bn = false; op.relu = false; }  // :117-120
    if (needs_bn && op.kind == 0) op.inorm[0] = add_in(net.get(), name + ".n", next, op.conv[0]);
    net->ops.push_back(op);
    prev = next;
  }
  FAV_REQUIRE(prev == 3, "the last layer must produce 3 channels (got %d)", prev);
  FAV_REQUIRE(net->ops.back().kind == 0 && !net->convs[net->ops.back().conv[0]].transposed,
              "the last arch token must be a (non-transposed) convolution");
  if (scale != 1.0) {  // the final layer writes a [3][H][W] frame: a net that resizes the frame would write past it
    set_error("arch '%s' resizes the frame by %g (its strided and upsampling layers must cancel)", arch, 1.0 / scale);
    return FAV_ERR_UNSUPPORTED;
  }
  for (ConvDef &c : net->convs) c.raw_out = &c != &net->convs[net->ops.back().conv[0]];  // only the last may x-fold
  FAV_REQUIRE(shrink == std::floor(shrink) && ((int)shrink) % 2 == 0, "unsupported shrink %f", shrink);
  net->reflect_pad = (int)shrink / 2;  // train_video.lua:319-324
  *out = net.release();
  return FAV_OK;
}

void fav_net_destroy(fav_net_t *net) { delete net; }

int fav_net_num_params(const fav_net_t *net) { return net ? (int)net->params.size() : 0; }

int fav_net_param_info(const fav_net_t *net, int index, char *name_out, int64_t shape_out[4], int64_t *numel) {
  FAV_REQUIRE(net && index >= 0 && index < (int)net->params.size(), "fav_net_param_info: bad index");
  const Param &p = net->params[index];
  if (name_out) { strncpy(name_out, p.name.c_str(), 63); name_out[63] = 0; }
  if (shape_out) for (int i = 0; i < 4; ++i) shape_out[i] = p.shape[i];
  if (numel) *numel = p.numel;
  return FAV_OK;
}

int fav_net_set_param(fav_net_t *net, const char *name, const float *host_data, int64_t numel) {
  FAV_REQUIRE(net && name && host_data, "fav_net_set_param: null argument");
  FAV_REQUIRE(!net->finalized, "fav_net_set_param: net already finalized");
  for (Param &p : net->params)
    if (p.name == name) {
      FAV_REQUIRE(numel == p.numel, "param %s: expected %lld elements, got %lld", name, (long long)p.numel,
                  (long long)numel);
      p.host.assign(host_data, host_data + numel);
      p.set = true;
      return FAV_OK;
    }
  set_error("fav_net_set_param: unknown parameter '%s'", name);
  return FAV_ERR_INVALID;
}

int fav_net_finalize(fav_net_t *net) {
  FAV_REQUIRE(net, "fav_net_finalize: null net");
  if (net->finalized) return FAV_OK;
  for (Param &p : net->params) FAV_REQUIRE(p.set, "fav_net_finalize: parameter %s was never set", p.name.c_str());
  std::vector<std::vector<float>> cw, cb, cs;
  FAV_TRY(fold_batch_norms(net, cw, cb, cs));
  // K-step tables (N blocks for Cout > 128) of every convolution, before any device work: a layer the tensor-core path
  // cannot run is refused here, by name, rather than at the first forward
  for (ConvDef &c : net->convs) {
    FAV_TRY(plan_conv_nblocks(c));
    if (!net->bn) FAV_TRY(plan_phase_stack(c));  // a batch-normalized net's operand epilogue runs one phase per job
  }
  FAV_TRY(require_device());
  cudaDeviceProp prop;
  FAV_TRY(check_cuda(cudaGetDevice(&net->device), "cudaGetDevice"));
  FAV_TRY(check_cuda(cudaGetDeviceProperties(&prop, net->device), "cudaGetDeviceProperties"));
  if (prop.major != 9) {
    set_error("libfav_b200 targets sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
    return FAV_ERR_UNSUPPORTED;
  }
  net->num_sms = prop.multiProcessorCount;
  for (size_t i = 0; i < net->convs.size(); ++i)
    FAV_TRY(pack_conv_weights(net, net->convs[i], net->params[net->convs[i].pw].host, cb[i], cw[i], cs[i]));
  for (InDef &n : net->inorms) {
    FAV_TRY(dev_upload(net, net->params[n.pw].host, &n.d_gamma));
    FAV_TRY(dev_upload(net, net->params[n.pb].host, &n.d_beta));
    if (!n.h_scale.empty()) {
      FAV_TRY(dev_upload(net, n.h_mean, &n.d_mean));
      FAV_TRY(dev_upload(net, n.h_scale, &n.d_scale));
    }
  }
  net->finalized = true;
  return FAV_OK;
}

int fav_net_set_conv_impl(fav_net_t *net, int impl) {
  FAV_REQUIRE(net && (impl == 0 || impl == 1), "fav_net_set_conv_impl: impl must be 0 (tcgen05) or 1 (CUDA cores)");
  net->conv_impl = impl;
  return FAV_OK;
}

// The plans (and their CUDA graphs) hold jobs built for one precision: switching drops them, and the next call rebuilds.
int fav_net_set_precision(fav_net_t *net, const char *mode) {
  FAV_REQUIRE(net && mode, "fav_net_set_precision: null argument");
  int single;
  if (!strcmp(mode, "pair")) single = 0;
  else if (!strcmp(mode, "fp16")) single = 1;
  else {
    set_error("fav_net_set_precision: mode \"%s\": \"pair\" (exact fp32 parity) or \"fp16\" (single pass)", mode);
    return FAV_ERR_INVALID;
  }
  if (single == net->single) return FAV_OK;
  net->plans.clear();
  net->last_plan = nullptr;
  net->single = single;
  return FAV_OK;
}

// Every device parameter buffer of a finalized net, in one fixed order (null where the net has no such buffer): the
// buffers a style bank holds one copy of per style
static std::vector<void **> bank_slots(fav_net *net) {
  std::vector<void **> v;
  auto add = [&v](auto *&p) { v.push_back(reinterpret_cast<void **>(&p)); };
  for (ConvDef &c : net->convs) {
    add(c.d_bias); add(c.d_scale); add(c.d_stack_bias);
    for (ConvPhase &ph : c.phases) { add(ph.d_w_simt); add(ph.d_b_tc); }
    for (ConvPhase &ph : c.stack) add(ph.d_b_tc);
    for (ConvDef &cb : c.nblock) {
      add(cb.d_bias); add(cb.d_scale);
      for (ConvPhase &ph : cb.phases) add(ph.d_b_tc);
    }
  }
  for (InDef &n : net->inorms) { add(n.d_gamma); add(n.d_beta); add(n.d_mean); add(n.d_scale); }
  return v;
}

// Style S of net = style 0 of src: each bank buffer grows by one copy of src's (a new allocation: the S styles it held, then
// src's), every pointer of the net moves to its new bank, and the plans built for S styles are dropped.
int fav_net_add_style(fav_net_t *net, const fav_net_t *src, int *index_out) {
  FAV_REQUIRE(net && src && index_out, "fav_net_add_style: null argument");
  FAV_REQUIRE(net->finalized && src->finalized, "fav_net_add_style: both nets must be finalized (fav_net_finalize)");
  FAV_REQUIRE(net != src, "fav_net_add_style: a net cannot add itself");
  FAV_REQUIRE(net->arch == src->arch, "fav_net_add_style: the nets differ in arch ('%s' and '%s')", net->arch.c_str(), src->arch.c_str());
  FAV_REQUIRE(net->padding_type == src->padding_type, "fav_net_add_style: the nets differ in padding_type ('%s' and '%s')",
              net->padding_type.c_str(), src->padding_type.c_str());
  FAV_REQUIRE(net->tanh_c == src->tanh_c, "fav_net_add_style: the nets differ in tanh_constant (%g and %g)", net->tanh_c, src->tanh_c);
  FAV_REQUIRE(net->in_dim == src->in_dim, "fav_net_add_style: the nets differ in in_dim (%d and %d)", net->in_dim, src->in_dim);
  FAV_REQUIRE(net->bn == src->bn, "fav_net_add_style: the nets differ in norm ('%s' and '%s')", net->bn ? "batch" : "instance",
              src->bn ? "batch" : "instance");
  FAV_REQUIRE(net->device == src->device, "fav_net_add_style: the nets live on devices %d and %d", net->device, src->device);
  FAV_REQUIRE(net->nstyles < kMaxBatch, "fav_net_add_style: a net holds at most %d styles (the batch limit)", kMaxBatch);
  const int S = net->nstyles;
  if (net->d_unscale.empty()) {
    for (const ConvDef &c : net->convs) {
      float *d = nullptr;
      FAV_TRY(check_cuda(cudaMalloc(&d, kMaxBatch * sizeof(float)), "cudaMalloc(style unscale)"));
      net->allocs.push_back(d);
      net->d_unscale.push_back(d);
      const float u = ldexpf(1.f, -c.w_exp);
      FAV_TRY(check_cuda(cudaMemcpy(d, &u, sizeof(float), cudaMemcpyHostToDevice), "cudaMemcpy(style unscale)"));
    }
  }
  std::vector<void **> to = bank_slots(net), from = bank_slots(const_cast<fav_net *>(src));
  // allocate every grown bank first: a failure leaves the net as it was
  std::vector<void *> grown(to.size(), nullptr);
  int rc = FAV_OK;
  for (size_t i = 0; i < to.size() && rc == FAV_OK; ++i) {
    if ((*to[i] == nullptr) != (*from[i] == nullptr) || (*to[i] && net->bank.at(*to[i]) != src->bank.at(*from[i]))) {
      set_error("fav_net_add_style: internal: parameter buffer %zu differs in size", i);
      rc = FAV_ERR_INVALID;
    } else if (*to[i]) {
      rc = check_cuda(cudaMalloc(&grown[i], (S + 1) * net->bank.at(*to[i])), "cudaMalloc(style bank)");
    }
  }
  for (size_t i = 0; i < to.size() && rc == FAV_OK; ++i) {
    if (!*to[i]) continue;
    const size_t per = net->bank.at(*to[i]);
    rc = check_cuda(cudaMemcpy(grown[i], *to[i], S * per, cudaMemcpyDeviceToDevice), "cudaMemcpy(style bank)");
    if (rc == FAV_OK)
      rc = check_cuda(cudaMemcpy((char *)grown[i] + S * per, *from[i], per, cudaMemcpyDeviceToDevice), "cudaMemcpy(style bank)");
  }
  for (size_t c = 0; c < net->convs.size() && rc == FAV_OK; ++c) {
    const float u = ldexpf(1.f, -src->convs[c].w_exp);
    rc = check_cuda(cudaMemcpy(net->d_unscale[c] + S, &u, sizeof(float), cudaMemcpyHostToDevice), "cudaMemcpy(style unscale)");
  }
  if (rc != FAV_OK) {
    for (void *p : grown) cudaFree(p);
    return rc;
  }
  net->plans.clear();
  net->last_plan = nullptr;
  for (size_t i = 0; i < to.size(); ++i) {
    if (!*to[i]) continue;
    const size_t per = net->bank.at(*to[i]);
    net->bank.erase(*to[i]);
    net->allocs.erase(std::find(net->allocs.begin(), net->allocs.end(), *to[i]));
    cudaFree(*to[i]);
    *to[i] = grown[i];
    net->bank[grown[i]] = per;
    net->allocs.push_back(grown[i]);
  }
  net->nstyles = S + 1;
  *index_out = S;
  return FAV_OK;
}

int fav_net_num_styles(const fav_net_t *net) { return net ? net->nstyles : 0; }

int fav_net_set_batch_styles(fav_net_t *net, const int *styles, int n) {
  FAV_REQUIRE(net && (n == 0 || styles), "fav_net_set_batch_styles: null argument");
  FAV_REQUIRE(n >= 0 && n <= kMaxBatch, "fav_net_set_batch_styles: %d entries; a batch has 1 to %d frames (0 clears)", n, kMaxBatch);
  for (int i = 0; i < n; ++i)
    FAV_REQUIRE(styles[i] >= 0 && styles[i] < net->nstyles, "fav_net_set_batch_styles: image %d gets style %d; the net holds %d",
                i, styles[i], net->nstyles);
  net->batch_styles.assign(styles, styles + n);
  return FAV_OK;
}

int fav_net_set_activation_budget(fav_net_t *net, size_t bytes) {
  FAV_REQUIRE(net && bytes > 0, "fav_net_set_activation_budget: null net or zero budget");
  net->budget = bytes;
  return FAV_OK;
}

int fav_net_plan_bytes(fav_net_t *net, int B, int H, int W, size_t *all_live, size_t *shared) {
  FAV_REQUIRE(net && all_live && shared, "fav_net_plan_bytes: null argument");
  FAV_REQUIRE(net->finalized, "fav_net_plan_bytes: call fav_net_finalize first");
  FAV_REQUIRE(B >= 1 && B <= kMaxBatch, "batch of %d frames: 1 to %d frames per call", B, kMaxBatch);
  FAV_REQUIRE(H % 4 == 0 && W % 4 == 0 && H >= 16 && W >= 16, "frame size %dx%d: H and W must be multiples of 4 and at least 16",
              W, H);
  return plan_sizes(net, B, H, W, all_live, shared);
}

int fav_net_forward(fav_net_t *net, const float *in7, int H, int W, float *out3, void *stream) {
  return fav_net_forward_batch(net, in7, 1, H, W, out3, stream);
}

int fav_net_forward_batch(fav_net_t *net, const float *in, int B, int H, int W, float *out3, void *stream) {
  FAV_REQUIRE(net && in && out3, "fav_net_forward: null argument");
  FAV_REQUIRE(net->finalized, "fav_net_forward: call fav_net_finalize first");
  Plan *pl;
  FAV_TRY(plan_for_call(net, B, H, W, (cudaStream_t)stream, &pl));
  return run_plan(net, *pl, in, out3, 1, (cudaStream_t)stream);
}

int fav_net_profile(fav_net_t *net, const float *in7, int H, int W, float *out3, int max_steps, int *kinds, float *ms,
                    double *work, char *names24, int *n_out, void *stream) {
  FAV_REQUIRE(net && in7 && out3 && kinds && ms && work && n_out, "fav_net_profile: null argument");
  FAV_REQUIRE(net->finalized, "fav_net_profile: call fav_net_finalize first");
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, 1, H, W, st, &pl));
  std::vector<ProfRec> prof;
  int rc = run_plan(net, *pl, in7, out3, 1, st, &prof);
  if (rc == FAV_OK) rc = check_cuda(cudaStreamSynchronize(st), "fav_net_profile sync");
  int n = 0;
  for (ProfRec &r : prof) {
    if (rc == FAV_OK && n < max_steps) {
      cudaEventElapsedTime(&r.ms, r.e0, r.e1);
      kinds[n] = r.kind; ms[n] = r.ms; work[n] = r.work;
      if (names24) memcpy(names24 + 24 * n, r.name, 24);
      ++n;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  *n_out = n;
  return rc;
}

int fav_net_layer_output(fav_net_t *net, int index, float *out, int *C, int *Hl, int *Wl, void *stream) {
  return fav_net_layer_output_image(net, index, 0, out, C, Hl, Wl, stream);
}

int fav_net_layer_output_image(fav_net_t *net, int index, int b, float *out, int *C, int *Hl, int *Wl, void *stream) {
  FAV_REQUIRE(net && net->last_plan, "fav_net_layer_output: run a forward first");
  Plan *pl = net->last_plan;
  FAV_REQUIRE(b >= 0 && b < pl->B, "fav_net_layer_output: image %d of a batch of %d", b, pl->B);
  auto it = pl->layer_operand.find(index);
  FAV_REQUIRE(it != pl->layer_operand.end(), "fav_net_layer_output: layer %d has no stored activation", index);
  const Operand &o = pl->ops[it->second];
  if (pl->arena) {  // operands share buffers: a later layer may have taken this one over, and a replay would clobber others
    bool fused = false;
    for (const PlanStep &s : pl->steps) fused |= s.layer_index == index && s.kind == 1 && s.fused_nl && net->conv_impl == 0;
    FAV_REQUIRE(pl->kept[it->second] && !fused, "fav_net_layer_output: layer %d of the %dx%d plan (batch of %d) is not kept: "
                "its activations share buffers with later layers (fav_net_set_activation_budget)", index, pl->W, pl->H, pl->B);
  }
  if (C) *C = o.C;
  if (Hl) *Hl = o.H;
  if (Wl) *Wl = o.W;
  if (!out) return FAV_OK;
  // a pass folded into its consumer (norm-on-load) never wrote this operand: replay the forward up to it with the pass run.
  // The replay starts from the net's first operand, which the forward leaves intact, so it recomputes the same bits.
  for (size_t si = 0; si < pl->steps.size(); ++si) {
    const PlanStep &s = pl->steps[si];
    if (s.layer_index == index && s.kind == 1 && s.fused_nl && net->conv_impl == 0) {
      FAV_TRY(run_plan(net, *pl, nullptr, nullptr, 1, (cudaStream_t)stream, nullptr, (int)si, true));
      break;
    }
  }
  return launch_unpack_operand(image_of(o, b), out, (cudaStream_t)stream);
}

int fav_run_image(fav_net_t *net, const float *content, const float *fill, int H, int W, float *out_rgb,
                  void *stream) {
  return fav_run_image_batch(net, content, fill, 1, H, W, out_rgb, stream);
}

int fav_run_image_batch(fav_net_t *net, const float *content, const float *fill, int B, int H, int W, float *out_rgb,
                        void *stream) {
  FAV_REQUIRE(net && content && out_rgb, "fav_run_image: null argument");
  FAV_REQUIRE(net->finalized, "fav_run_image: call fav_net_finalize first");
  // model_img == nil: the video model on cat(pre(img), fill, zeros) (core.lua:133-138); a separate 3-channel image model
  // (-model_img, core.lua:61-68,146) gets pre(img) only -- the same fused input kernel, whose channels 3..7 are then zero
  FAV_REQUIRE(net->in_dim == 7 || net->in_dim == 3, "fav_run_image: video model (7 input channels) or image model (3) required");
  if (net->in_dim == 3) fill = nullptr;
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, B, H, W, st, &pl));
  static const bool fuse_pack = getenv("FAV_NO_FUSEPACK") == nullptr;
  if (fuse_pack) {
    FAV_TRY(launch_temporal_input_packed(content, nullptr, nullptr, nullptr, fill, nullptr, pl->ops[0], net->reflect_pad, H, W, 0, true, st,
                                         B));
    return run_plan_frame(net, *pl, nullptr, out_rgb, st);
  }
  FAV_TRY(launch_temporal_input(content, nullptr, nullptr, nullptr, fill, nullptr, pl->in7, H, W, 0, true, st, B));
  return run_plan_frame(net, *pl, pl->in7, out_rgb, st);  // deprocess fused into the last epilogue (core.lua:149)
}

// a-9 with -scale_factor (core.lua:127-130,146-152): image.scale(img, W*sf, H*sf, 'bicubic') -> model_img(pre(.)) ->
// deprocess -> image.scale(., W, H, 'bicubic').  The network runs at h x w on the (1, h, w) plan, into the plan's own out3,
// so the plan keeps one cached graph however many destinations the caller cycles through.
int fav_run_image_scaled(fav_net_t *net, const float *content, int H, int W, double scale_factor, float *out_rgb, void *stream) {
  if (scale_factor == 1.0) return fav_run_image(net, content, nullptr, H, W, out_rgb, stream);
  FAV_REQUIRE(net && content && out_rgb, "fav_run_image_scaled: null argument");
  FAV_REQUIRE(net->finalized, "fav_run_image_scaled: call fav_net_finalize first");
  // model_img == nil: the reference concatenates the scaled frame with a fill of the unscaled size, and torch.cat fails
  FAV_REQUIRE(net->in_dim == 3, "fav_run_image_scaled: -scale_factor %g needs a separate image model (3 input channels); the "
              "video model's input joins the scaled frame with an unscaled fill (fast_artistic_video_core.lua:133-138)", scale_factor);
  const double hd = H * scale_factor, wd = W * scale_factor;
  FAV_REQUIRE(std::isfinite(scale_factor) && scale_factor > 0 && hd == std::floor(hd) && wd == std::floor(wd) && hd < 1e9 &&
                  wd < 1e9,
              "fav_run_image_scaled: %dx%d at -scale_factor %g is %gx%g; the scaled frame needs integer sides (image.scale, then "
              "view(1, 3, H*sf, W*sf), fast_artistic_video_core.lua:128-130)", W, H, scale_factor, wd, hd);
  const int h = (int)hd, w = (int)wd;
  FAV_TRY(check_scale_args(content, out_rgb, 3, H, W, h, w));
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, 1, h, w, st, &pl));  // the frame rules apply at h x w; refusals come before any device work
  // not pl->in7: fav_run_image's unfused path (FAV_NO_FUSEPACK) writes that one
  if (!pl->scaled_in) FAV_TRY(alloc_zero(*pl, (void **)&pl->scaled_in, (size_t)3 * h * w * sizeof(float)));
  FAV_TRY(launch_image_scale_bicubic(content, pl->scaled_in, 3, H, W, h, w, st));
  FAV_TRY(launch_temporal_input_packed(pl->scaled_in, nullptr, nullptr, nullptr, nullptr, nullptr, pl->ops[0], net->reflect_pad, h, w,
                                       0, true, st));
  FAV_TRY(run_plan_frame(net, *pl, nullptr, pl->out3, st));
  return launch_image_scale_bicubic(pl->out3, out_rgb, 3, h, w, H, W, st);  // unclamped, like the reference's img_out
}

int fav_run_next_image(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow,
                       const float *cert, const float *fill, const float *flow_mask, int H, int W, int border_mode,
                       float *out_rgb, void *stream) {
  return fav_run_next_image_batch(net, content, prev_rgb, flow, cert, fill, flow_mask, 1, H, W, border_mode, out_rgb, stream);
}

int fav_run_next_image_batch(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow,
                             const float *cert, const float *fill, const float *flow_mask, int B, int H, int W, int border_mode,
                             float *out_rgb, void *stream) {
  FAV_REQUIRE(net && content && prev_rgb && flow && cert && out_rgb, "fav_run_next_image: null argument");
  FAV_REQUIRE(net->finalized, "fav_run_next_image: call fav_net_finalize first");
  FAV_REQUIRE(net->in_dim == 7, "fav_run_next_image: video model (7 input channels) required");
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, B, H, W, st, &pl));
  static const bool fuse_pack = getenv("FAV_NO_FUSEPACK") == nullptr;
  if (fuse_pack) {
    FAV_TRY(launch_temporal_input_packed(content, prev_rgb, flow, cert, fill, flow_mask, pl->ops[0], net->reflect_pad, H, W,
                                         border_mode, false, st, B));
    return run_plan_frame(net, *pl, nullptr, out_rgb, st);
  }
  FAV_TRY(launch_temporal_input(content, prev_rgb, flow, cert, fill, flow_mask, pl->in7, H, W, border_mode, false, st, B));
  return run_plan_frame(net, *pl, pl->in7, out_rgb, st);  // core.lua:172-173
}

// a-8 with the certainty computed inside: the whole temporal stage (occlusion test or given certainty -> min filter -> warp
// -> preprocess -> mask -> concat) is ONE kernel that writes the network's first operand, followed by one graph launch.
int fav_run_next_image_flows(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow_bw,
                             const float *flow_fw_uv, const float *cert_raw, const float *fill, const float *flow_mask,
                             int H, int W, int min_filter_r, int border_mode, float *out_rgb, void *stream) {
  return fav_run_next_image_flows_batch(net, content, prev_rgb, flow_bw, flow_fw_uv, cert_raw, fill, flow_mask, 1, H, W,
                                        min_filter_r, border_mode, out_rgb, stream);
}

int fav_run_next_image_flows_batch(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow_bw,
                                   const float *flow_fw_uv, const float *cert_raw, const float *fill, const float *flow_mask,
                                   int B, int H, int W, int min_filter_r, int border_mode, float *out_rgb, void *stream) {
  FAV_REQUIRE(net && content && prev_rgb && flow_bw && out_rgb, "fav_run_next_image_flows: null argument");
  FAV_REQUIRE((flow_fw_uv != nullptr) != (cert_raw != nullptr), "fav_run_next_image_flows: give either the forward flow or a certainty plane");
  FAV_REQUIRE(net->finalized, "fav_run_next_image_flows: call fav_net_finalize first");
  FAV_REQUIRE(net->in_dim == 7, "fav_run_next_image_flows: video model (7 input channels) required");
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  FAV_REQUIRE(min_filter_r >= 0 && (min_filter_r <= 1 || (min_filter_r & 1)) && min_filter_r <= 15, "occlusions_min_filter must be odd <= 15");
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, B, H, W, st, &pl));
  static const bool no_stage = getenv("FAV_NO_STAGE") != nullptr;  // A/B timing: the three separate kernels
  int rc = no_stage ? FAV_ERR_UNSUPPORTED
                    : launch_temporal_stage(content, prev_rgb, flow_bw, flow_fw_uv, cert_raw, fill, flow_mask, nullptr, nullptr,
                                            &pl->ops[0], net->reflect_pad, H, W, min_filter_r, border_mode, st, B);
  if (rc == FAV_ERR_UNSUPPORTED) {  // unaligned planes / W % 4 != 0: the three separate kernels
    const int64_t HW = (int64_t)H * W;
    if (!pl->cert_a) {
      FAV_TRY(alloc_zero(*pl, (void **)&pl->cert_a, B * HW * sizeof(float)));
      FAV_TRY(alloc_zero(*pl, (void **)&pl->cert_b, B * HW * sizeof(float)));
    }
    const float *cert = cert_raw;
    if (flow_fw_uv) {
      for (int b = 0; b < B; ++b) {
        const float *bw = flow_bw + 2 * b * HW, *fw = flow_fw_uv + 2 * b * HW;
        FAV_TRY(launch_consistency(bw + HW, bw, fw, fw + HW, nullptr, nullptr, 0.f, nullptr, pl->cert_a + b * HW, W, H, st));
      }
      cert = pl->cert_a;
    }
    if (min_filter_r > 1) {
      FAV_TRY(launch_min_filter(cert, pl->cert_b, B, H, W, min_filter_r, st));
      cert = pl->cert_b;
    }
    rc = launch_temporal_input_packed(content, prev_rgb, flow_bw, cert, fill, flow_mask, pl->ops[0], net->reflect_pad, H, W,
                                      border_mode, false, st, B);
  }
  FAV_TRY(rc);
  return run_plan_frame(net, *pl, nullptr, out_rgb, st);
}

// a-8 in 4-argument mode (makeOptFlow_deepflow.sh:58-60, consistencyChecker.cpp:39-78,122-124,154-160): the certainty of
// fav_run_next_image_flows with the structure term of the frame being stylized.  `content` is image.load's byte/255, and
// fl(fl(byte/255) * 255) == byte, so the corners read CTensor's 0..255 planes of the same file.  Per frame: the corners chain,
// the fused stage (MODE 2), the network's graph launch.
int fav_run_next_image_flows_structure(fav_net_t *net, const float *content, const float *prev_rgb, const float *flow_bw,
                                       const float *flow_fw_uv, const float *fill, const float *flow_mask, int H, int W,
                                       int min_filter_r, int border_mode, float *out_rgb, void *stream) {
  FAV_REQUIRE(net && content && prev_rgb && flow_bw && flow_fw_uv && out_rgb, "fav_run_next_image_flows_structure: null argument");
  FAV_REQUIRE(net->finalized, "fav_run_next_image_flows_structure: call fav_net_finalize first");
  FAV_REQUIRE(net->in_dim == 7, "fav_run_next_image_flows_structure: video model (7 input channels) required");
  FAV_REQUIRE(H >= 3 && W >= 3, "fav_run_next_image_flows_structure: frame %dx%d below computeCorners' 3x3", W, H);
  FAV_REQUIRE(border_mode == FAV_BORDER_PER_TAP || border_mode == FAV_BORDER_PAD_PIXEL, "bad border_mode");
  FAV_REQUIRE(min_filter_r >= 0 && (min_filter_r <= 1 || (min_filter_r & 1)) && min_filter_r <= 15, "occlusions_min_filter must be odd <= 15");
  Plan *pl;
  cudaStream_t st = (cudaStream_t)stream;
  FAV_TRY(plan_for_call(net, 1, H, W, st, &pl));
  const int64_t HW = (int64_t)H * W;
  if (!pl->corners_ws) {
    FAV_TRY(alloc_zero(*pl, (void **)&pl->structure, HW * sizeof(float)));
    FAV_TRY(alloc_zero(*pl, (void **)&pl->structure_avg, 16));
    FAV_TRY(alloc_zero(*pl, &pl->corners_ws, fav_compute_corners_workspace(3, W, H)));
  }
  FAV_TRY(launch_compute_corners(content, 255.0f, 3, W, H, 3.0f, pl->structure, pl->structure_avg, pl->corners_ws, st));
  int rc = launch_temporal_stage_structure(content, prev_rgb, flow_bw, flow_fw_uv, pl->structure, pl->structure_avg, fill, flow_mask,
                                           nullptr, pl->ops[0], net->reflect_pad, H, W, min_filter_r, border_mode, st);
  if (rc == FAV_ERR_UNSUPPORTED) {  // unaligned planes / W % 4 != 0: the three separate kernels
    if (!pl->cert_a) {
      FAV_TRY(alloc_zero(*pl, (void **)&pl->cert_a, HW * sizeof(float)));
      FAV_TRY(alloc_zero(*pl, (void **)&pl->cert_b, HW * sizeof(float)));
    }
    FAV_TRY(launch_consistency(flow_bw + HW, flow_bw, flow_fw_uv, flow_fw_uv + HW, pl->structure, pl->structure_avg, 0.f, nullptr,
                               pl->cert_a, W, H, st));
    const float *cert = pl->cert_a;
    if (min_filter_r > 1) {
      FAV_TRY(launch_min_filter(cert, pl->cert_b, 1, H, W, min_filter_r, st));
      cert = pl->cert_b;
    }
    rc = launch_temporal_input_packed(content, prev_rgb, flow_bw, cert, fill, flow_mask, pl->ops[0], net->reflect_pad, H, W,
                                      border_mode, false, st);
  }
  FAV_TRY(rc);
  return run_plan_frame(net, *pl, nullptr, out_rgb, st);
}
}
