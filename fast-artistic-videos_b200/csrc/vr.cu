// vr.cu -- VR (cube-map) post-processing kernels, SURVEY.md §8 a-V / f-4:
//   median filter                 utils.median_filter            fast_artistic_video/utils.lua:151-159
//       (r x r windows by unfold, median over the r*r values = lower median, VALID region (H-r+1) x (W-r+1);
//        the reference round-trips to the CPU for it because CudaTensor has no median)
//   fused 4-way border blend      combineSides + blend           fast_artistic_video_vr.lua:146-152, 454-509
//       out = base * (1 - mask) + mask * sum_{i<4} warp(rot_i(side_i), map_i) / div
//       -- the reference runs 4 warp launches, 4 rotations (index copies), 4 divisions, 3 adds, 2 cmuls, 1 add per face;
//       here the rotation is an index mapping inside the gather and everything is one kernel.
//   -evaluate gradient metric     evaluate_gradient              fast_artistic_video_vr.lua:344-387
//       (the six double sums behind gradx / grady / gradmag: face gradients, max-pooled mask gradients and their products
//        in one pass over a shared-memory tile; the reference runs it on the CPU in double)
// Arithmetic follows the reference order with round-to-nearest intrinsics (bit-exact vs the oracle composition).
#include "fav_common.cuh"

namespace fav {

// ---- median ---------------------------------------------------------------------------------------------------
template <int R>
__global__ void __launch_bounds__(256) median_kernel(const float *__restrict__ in, float *__restrict__ out, int C, int H, int W) {
  const int Wo = W - R + 1, Ho = H - R + 1;
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, c = blockIdx.z;
  if (x >= Wo || y >= Ho) return;
  float v[R * R];
  const float *p = in + ((int64_t)c * H + y) * W + x;
#pragma unroll
  for (int dy = 0; dy < R; ++dy)
#pragma unroll
    for (int dx = 0; dx < R; ++dx) v[dy * R + dx] = __ldg(p + (int64_t)dy * W + dx);
  // partial selection sort up to the (lower) median index: torch.median returns element (n-1)/2 of the sorted values
  constexpr int N = R * R, K = (N - 1) / 2;
#pragma unroll
  for (int i = 0; i <= K; ++i) {
#pragma unroll
    for (int j = i + 1; j < N; ++j) {
      float a = v[i], b = v[j];
      v[i] = fminf(a, b);
      v[j] = fmaxf(a, b);
    }
  }
  out[((int64_t)c * Ho + y) * Wo + x] = v[K];
}

// ---- fused border blend -------------------------------------------------------------------------------------------
struct BlendSide {
  const float *img;   // [3,S,S] stylized neighbour face
  const float *map;   // [2,S,S] perspective warp map (dy,dx), sentinel 99999 outside the border strip
  int rot;            // 0 none, 1 rotate90, 2 rotateMinus90, 3 rotate180   (fast_artistic_video_vr.lua:134-144)
};
struct BlendArgs {
  BlendSide s[4];
  const float *base;      // [3,S,S]
  const float *div;       // [S,S] mask_all_div
  const float *mask;      // [S,S] blend mask (grad_mask_all)
  const float *anti;      // [S,S] 1 - grad_mask_all as the reference casts it from double (:456), or null
  float *out;             // [3,S,S]
  int S;
};

// value of rot(img)[c][y][x] for a square S x S face
__device__ __forceinline__ float rot_fetch(const float *__restrict__ img, int rot, int c, int y, int x, int S) {
  int sy, sx;
  if (rot == 0) { sy = y; sx = x; }
  else if (rot == 1) { sy = x; sx = S - 1 - y; }       // rotate90:      R[y][x] = t[x][S-1-y]
  else if (rot == 2) { sy = S - 1 - x; sx = y; }       // rotateMinus90: R[y][x] = t[S-1-x][y]
  else { sy = S - 1 - y; sx = S - 1 - x; }             // rotate180
  return __ldg(img + ((int64_t)c * S + sy) * S + sx);
}

__global__ void __launch_bounds__(256) vr_blend_kernel(const __grid_constant__ BlendArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int S = a.S;
  if (x >= S || y >= S) return;
  const int64_t o = (int64_t)y * S + x, SS = (int64_t)S * S;
  const float m = __ldg(a.mask + o), dv = __ldg(a.div + o);
  float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float dy = __ldg(a.s[i].map + o), dx = __ldg(a.s[i].map + SS + o);
    // bilinear sample exactly as BilinearSamplerBDHW.cu:72-108 (per-corner zero fill)
    float yf = __fadd_rn(dy, (float)y), xf = __fadd_rn(dx, (float)x);
    float fy = floorf(yf), fx = floorf(xf);
    int y0 = (int)fy, x0 = (int)fx;
    float wx = __fsub_rn(1.0f, __fsub_rn(xf, (float)x0)), wy = __fsub_rn(1.0f, __fsub_rn(yf, (float)y0));
    bool xin0 = x0 >= 0 && x0 <= S - 1, xin1 = x0 + 1 >= 0 && x0 + 1 <= S - 1;
    bool yin0 = y0 >= 0 && y0 <= S - 1, yin1 = y0 + 1 >= 0 && y0 + 1 <= S - 1;
    float omx = __fsub_rn(1.0f, wx), omy = __fsub_rn(1.0f, wy);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float vtl = (xin0 && yin0) ? rot_fetch(a.s[i].img, a.s[i].rot, c, y0, x0, S) : 0.f;
      float vtr = (xin1 && yin0) ? rot_fetch(a.s[i].img, a.s[i].rot, c, y0, x0 + 1, S) : 0.f;
      float vbl = (xin0 && yin1) ? rot_fetch(a.s[i].img, a.s[i].rot, c, y0 + 1, x0, S) : 0.f;
      float vbr = (xin1 && yin1) ? rot_fetch(a.s[i].img, a.s[i].rot, c, y0 + 1, x0 + 1, S) : 0.f;
      float v = bilinear_ref_blend(wx, wy, omx, omy, vtl, vtr, vbl, vbr);
      float q = __fdiv_rn(v, dv);                      // torch.cdiv(side, divisor)   (combineSides :147-151)
      acc[c] = i == 0 ? q : __fadd_rn(acc[c], q);
    }
  }
  const float am = a.anti ? __ldg(a.anti + o) : __fsub_rn(1.0f, m);  // anti_mask = 1 - grad_mask_all  (:456)
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float b = __ldg(a.base + c * SS + o);
    a.out[c * SS + o] = __fadd_rn(__fmul_rn(b, am), __fmul_rn(acc[c], m));  // :466
  }
}

// ---- -evaluate gradient metric (evaluate_gradient, fast_artistic_video_vr.lua:344-387) -----------------------------
// One CTA per kEvTX x kEvTY tile of the H x W grid; thread t owns column x0 + t and walks the tile's rows.  Everything is in
// double from the fp32 inputs, as the reference computes after :double():
//   gx = max_c |f[c][y][x+2] - f[c][y][x]|  on [H, W-2]      gy = max_c |f[c][y+2][x] - f[c][y][x]|  on [H-2, W]
//   MX = 3x3 max-pool (stride 1, padding cells ignored) of |m[y][x+2] - m[y][x]| on [H, W-2], MY likewise on [H-2, W].
// The pool is separable: each row's 3-wide horizontal maximum is formed once and the vertical maximum slides over three of
// them in registers.  Out-of-domain cells enter as 0, which leaves the maximum of non-negative values unchanged.
// Sums: per thread in row order, per CTA by a fixed tree, then vr_eval_finish_kernel adds the CTA partials in tile order.
constexpr int kEvTX = 128, kEvTY = 16;

__global__ void __launch_bounds__(kEvTX) vr_eval_gradient_kernel(const float *__restrict__ face, const float *__restrict__ mask,
                                                                 int H, int W, double *__restrict__ part) {
  __shared__ float sf[3][kEvTY + 2][kEvTX + 2];  // face rows y0 .. y0+TY+1, columns x0 .. x0+TX+1
  __shared__ float sm[kEvTY + 4][kEvTX + 4];     // mask rows y0-1 .. y0+TY+2, columns x0-1 .. x0+TX+2
  __shared__ double red[kEvTX];
  const int x0 = blockIdx.x * kEvTX, y0 = blockIdx.y * kEvTY, t = threadIdx.x;
  const int64_t HW = (int64_t)H * W;
  for (int i = t; i < 3 * (kEvTY + 2) * (kEvTX + 2); i += kEvTX) {
    const int c = i / ((kEvTY + 2) * (kEvTX + 2)), r = i / (kEvTX + 2) % (kEvTY + 2), q = i % (kEvTX + 2);
    const int gy = y0 + r, gx = x0 + q;
    sf[c][r][q] = (gy < H && gx < W) ? __ldg(face + c * HW + (int64_t)gy * W + gx) : 0.f;
  }
  for (int i = t; i < (kEvTY + 4) * (kEvTX + 4); i += kEvTX) {
    const int r = i / (kEvTX + 4), q = i % (kEvTX + 4);
    const int gy = y0 - 1 + r, gx = x0 - 1 + q;
    sm[r][q] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(mask + (int64_t)gy * W + gx) : 0.f;
  }
  __syncthreads();

  const int x = x0 + t;
  // horizontal 3-maxima of |dm_x| (domain [H, W-2]) and |dm_y| (domain [H-2, W]) of global row gy, for this column
  auto hmax_x = [&](int gy) {
    double v = 0.0;
    if (gy < 0 || gy >= H) return v;
    const float *row = &sm[gy - y0 + 1][t + 1];  // row[d] = m[gy][x + d]
#pragma unroll
    for (int d = -1; d <= 1; ++d)
      if (x + d >= 0 && x + d < W - 2) v = fmax(v, fabs((double)row[d + 2] - (double)row[d]));
    return v;
  };
  auto hmax_y = [&](int gy) {
    double v = 0.0;
    if (gy < 0 || gy >= H - 2) return v;
    const float *r0 = &sm[gy - y0 + 1][t + 1], *r2 = &sm[gy - y0 + 3][t + 1];
#pragma unroll
    for (int d = -1; d <= 1; ++d)
      if (x + d >= 0 && x + d < W) v = fmax(v, fabs((double)r2[d] - (double)r0[d]));
    return v;
  };
  double s_gx = 0.0, s_gy = 0.0, s_mx = 0.0, s_my = 0.0, s_gxm = 0.0, s_gym = 0.0;
  if (x < W) {
    double ax = hmax_x(y0 - 1), bx = hmax_x(y0), ay = hmax_y(y0 - 1), by = hmax_y(y0);
    const int ye = min(kEvTY, H - y0);
    for (int r = 0; r < ye; ++r) {
      const int y = y0 + r;
      const double cx = hmax_x(y + 1), cy = hmax_y(y + 1);
      if (x < W - 2) {
        const double mx = fmax(fmax(ax, bx), cx);
        double g = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) g = fmax(g, fabs((double)sf[c][r][t + 2] - (double)sf[c][r][t]));
        s_gx += g;
        s_mx += mx;
        s_gxm += __dmul_rn(g, mx);  // cmul, then sum: the product is rounded on its own
      }
      if (y < H - 2) {
        const double my = fmax(fmax(ay, by), cy);
        double g = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) g = fmax(g, fabs((double)sf[c][r + 2][t] - (double)sf[c][r][t]));
        s_gy += g;
        s_my += my;
        s_gym += __dmul_rn(g, my);
      }
      ax = bx; bx = cx; ay = by; by = cy;
    }
  }
  const double v[6] = {s_gx, s_gy, s_mx, s_my, s_gxm, s_gym};
  const int64_t nt = (int64_t)gridDim.x * gridDim.y, b = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    red[t] = v[k];
    __syncthreads();
#pragma unroll
    for (int s = kEvTX / 2; s > 0; s >>= 1) {
      if (t < s) red[t] += red[t + s];
      __syncthreads();
    }
    if (t == 0) part[k * nt + b] = red[0];
    __syncthreads();
  }
}

// sums[k] = sum over tiles, in tile order, of part[k][tile]: CTA k adds row k
__global__ void __launch_bounds__(256) vr_eval_finish_kernel(const double *__restrict__ part, int64_t nt, double *__restrict__ sums) {
  __shared__ double red[256];
  const int t = threadIdx.x;
  double s = 0.0;
  for (int64_t i = t; i < nt; i += 256) s += part[blockIdx.x * nt + i];
  red[t] = s;
  __syncthreads();
#pragma unroll
  for (int k = 128; k > 0; k >>= 1) {
    if (t < k) red[t] += red[t + k];
    __syncthreads();
  }
  if (t == 0) sums[blockIdx.x] = red[0];
}

}  // namespace fav

using namespace fav;

extern "C" {

int fav_median_filter(const float *in, float *out, int C, int H, int W, int r, void *stream) {
  FAV_REQUIRE(in && out, "median_filter: null tensor");
  FAV_REQUIRE(r == 1 || r == 3 || r == 5, "median_filter: r must be 1, 3 or 5");
  FAV_REQUIRE(C > 0 && H >= r && W >= r, "median_filter: image smaller than the window");
  FAV_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  dim3 block(32, 8), grid(ceil_div(W - r + 1, 32), ceil_div(H - r + 1, 8), C);
  if (r == 1) median_kernel<1><<<grid, block, 0, st>>>(in, out, C, H, W);
  else if (r == 3) median_kernel<3><<<grid, block, 0, st>>>(in, out, C, H, W);
  else median_kernel<5><<<grid, block, 0, st>>>(in, out, C, H, W);
  return post_launch("median_filter");
}

int fav_vr_blend_sides(const float *base, const float *const sides[4], const float *const maps[4], const int rot[4],
                       const float *div, const float *mask, const float *anti_mask, float *out, int S, void *stream) {
  FAV_REQUIRE(base && sides && maps && rot && div && mask && out, "vr_blend_sides: null argument");
  FAV_REQUIRE(S > 1, "vr_blend_sides: empty face");
  BlendArgs a;
  for (int i = 0; i < 4; ++i) {
    FAV_REQUIRE(sides[i] && maps[i] && rot[i] >= 0 && rot[i] <= 3, "vr_blend_sides: bad side %d", i);
    a.s[i].img = sides[i]; a.s[i].map = maps[i]; a.s[i].rot = rot[i];
  }
  a.base = base; a.div = div; a.mask = mask; a.anti = anti_mask; a.out = out; a.S = S;
  FAV_TRY(require_device());
  dim3 block(32, 8), grid(ceil_div(S, 32), ceil_div(S, 8));
  vr_blend_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(a);
  return post_launch("vr_blend_sides");
}

int fav_vr_eval_gradient(const float *face, const float *mask, int H, int W, double *sums_dev, void *stream) {
  FAV_REQUIRE(face && mask && sums_dev, "vr_eval_gradient: null argument");
  FAV_REQUIRE(H >= 3 && W >= 3, "vr_eval_gradient: face %dx%d, need H, W >= 3", H, W);
  FAV_REQUIRE(ceil_div(H, kEvTY) <= 65535, "vr_eval_gradient: H %d too large", H);
  FAV_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(ceil_div(W, kEvTX), ceil_div(H, kEvTY));
  const int64_t nt = (int64_t)grid.x * grid.y;
  // the CTA partials live on the stream's own pool allocation, so concurrent calls on different streams never share them
  double *part = nullptr;
  FAV_TRY(check_cuda(cudaMallocAsync((void **)&part, (size_t)nt * 6 * sizeof(double), st), "vr_eval_gradient: partials"));
  vr_eval_gradient_kernel<<<grid, kEvTX, 0, st>>>(face, mask, H, W, part);
  int rc = post_launch("vr_eval_gradient");
  if (rc == FAV_OK) {
    vr_eval_finish_kernel<<<6, 256, 0, st>>>(part, nt, sums_dev);
    rc = post_launch("vr_eval_gradient finish");
  }
  const int rf = check_cuda(cudaFreeAsync(part, st), "vr_eval_gradient: free partials");
  return rc != FAV_OK ? rc : rf;
}
}
