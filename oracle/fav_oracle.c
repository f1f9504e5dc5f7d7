/*
 * fav_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C, single-file CPU restatement of the reference's temporal-consistency
 * hot path (manuelruder/fast-artistic-videos @ bf1d072).  Every function cites
 * the reference file:line it follows.  It is the checker the CUDA product path
 * is compared against; nothing outside tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.
 *
 * Pinning status:
 *   - orc_check_consistency / orc_compute_corners / PGM+PPM+.flo I/O are pinned
 *     bit-for-bit against the reference's own consistencyChecker binary, which
 *     oracle/Makefile compiles unmodified into oracle/_ref/ (see
 *     tests/test_oracle_pinning.py and tests/golden/).
 *   - orc_warp_bdhw restates stnbdhw/BilinearSamplerBDHW.cu:13-32,58-108 line
 *     by line, including the FMA contraction nvcc applies to :103-106.  Pinned: the
 *     reference's kernel body, extracted from /root/reference at build time and
 *     compiled for sm_90a by oracle/Makefile (oracle/_ref/libref_warp.so), is
 *     bit-identical to the CUDA product on the GPU box (tests/test_gpu_refwarp.py),
 *     and its outputs on seeded inputs are committed as tests/golden/warp_ref_*.npz,
 *     which this restatement reproduces bit for bit (tests/test_oracle.py).
 *   - vgg pre/deprocess, min_filter, temporal-input assembly restate Lua code
 *     whose arithmetic lives in un-vendored, unpinned Torch7 rocks
 *     ("parity unpinned" at those third-party boundaries; see DESIGN.md).
 *   - orc_image_warp_pad restates third-party image.warp from its published
 *     algorithm: PARITY UNPINNED.
 *
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* a-1  nn.BilinearSamplerBDHW forward                                        */
/* stnbdhw/BilinearSamplerBDHW.cu:48-109 (kernel), :13-32 (helpers)           */
/* ------------------------------------------------------------------------- */

/* BilinearSamplerBDHW.cu:13-23 */
static inline void orc_get_top_left(float x, int *point, float *weight) {
  *point = (int)floor(x);                 /* :21 (double floor of a float)    */
  *weight = 1 - (x - *point);             /* :22 float arithmetic             */
}

/* BilinearSamplerBDHW.cu:25-28 */
static inline int orc_between(int v, int lo, int hi) { return v >= lo && v <= hi; }

/*
 * img   : B x C x Hin x Win, element strides is[4]
 * grid  : B x 2 x Hout x Wout (channel 0 = dy, 1 = dx; pixel offsets), gs[4]
 * out   : B x C x Hout x Wout, os[4]
 * Arithmetic order is that of BilinearSamplerBDHW.cu:72-108 (fp32; blend contracted as the compiled kernel).
 */
ORC_API void orc_warp_bdhw(const float *img, const int64_t is[4], const float *grid,
                           const int64_t gs[4], float *out, const int64_t os[4], int B,
                           int C, int Hin, int Win, int Hout, int Wout, int threads) {
  (void)threads;
#pragma omp parallel for collapse(2) num_threads(threads > 0 ? threads : 1) schedule(static)
  for (int b = 0; b < B; ++b)
    for (int yOut = 0; yOut < Hout; ++yOut)
      for (int xOut = 0; xOut < Wout; ++xOut) {
        /* :72-73 */
        float yf = grid[b * gs[0] + 0 * gs[1] + yOut * gs[2] + xOut * gs[3]] + yOut;
        float xf = grid[b * gs[0] + 1 * gs[1] + yOut * gs[2] + xOut * gs[3]] + xOut;
        int y0, x0;
        float wy, wx;
        orc_get_top_left(xf, &x0, &wx); /* :77 */
        orc_get_top_left(yf, &y0, &wy); /* :78 */
        /* :92-95 */
        int tl = orc_between(x0, 0, Win - 1) && orc_between(y0, 0, Hin - 1);
        int tr = orc_between(x0 + 1, 0, Win - 1) && orc_between(y0, 0, Hin - 1);
        int bl = orc_between(x0, 0, Win - 1) && orc_between(y0 + 1, 0, Hin - 1);
        int br = orc_between(x0 + 1, 0, Win - 1) && orc_between(y0 + 1, 0, Hin - 1);
        for (int ch = 0; ch < C; ++ch) {
          const float *p = img + b * is[0] + ch * is[1];
          float vtl = 0, vtr = 0, vbl = 0, vbr = 0; /* :86-90 */
          if (tl) vtl = p[(int64_t)y0 * is[2] + (int64_t)x0 * is[3]];             /* :98 */
          if (tr) vtr = p[(int64_t)y0 * is[2] + (int64_t)(x0 + 1) * is[3]];       /* :99 */
          if (bl) vbl = p[(int64_t)(y0 + 1) * is[2] + (int64_t)x0 * is[3]];       /* :100 */
          if (br) vbr = p[(int64_t)(y0 + 1) * is[2] + (int64_t)(x0 + 1) * is[3]]; /* :101 */
          /* :103-106 as nvcc contracts it (12.9, default -fmad=true, sm_90a; SASS of the reference kernel body:
           * FMUL,FMUL,FMUL,FFMA,FMUL,FMUL,FFMA,FFMA): the TR product is rounded, the other three terms are fused
           * into the running sum.  Pinned against the compiled reference kernel (oracle/ref_warp, tests/golden/warp_ref_*). */
          float omx = 1 - wx, omy = 1 - wy;
          float v = (omx * wy) * vtr;
          v = fmaf(wx * wy, vtl, v);
          v = fmaf(wx * omy, vbl, v);
          v = fmaf(omx * omy, vbr, v);
          out[b * os[0] + ch * os[1] + yOut * os[2] + xOut * os[3]] = v; /* :108 */
        }
      }
}

/*
 * a-1'  CPU branch of utils.warp_image: image.warp(img, flow,'bilinear',true,'pad',0)
 * (fast_artistic_video/utils.lua:145-147).  The arithmetic is in the third-party
 * torch `image` rock (not vendored, unpinned).  Restated from its published
 * algorithm: a pixel whose source coordinate lies outside [0,W-1]x[0,H-1] takes
 * the pad value as a whole; otherwise the 4 neighbours are index-clamped.
 * PARITY UNPINNED.
 */
ORC_API void orc_image_warp_pad(const float *img, const float *flow, float *out, int C, int H,
                                int W, float pad) {
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float iy = flow[(int64_t)0 * H * W + (int64_t)y * W + x] + y;
      float ix = flow[(int64_t)1 * H * W + (int64_t)y * W + x] + x;
      int off = (iy < 0 || iy > H - 1 || ix < 0 || ix > W - 1);
      for (int c = 0; c < C; ++c) {
        float v;
        if (off) {
          v = pad;
        } else {
          int y0 = (int)floorf(iy), x0 = (int)floorf(ix);
          int y1 = y0 + 1 > H - 1 ? H - 1 : y0 + 1;
          int x1 = x0 + 1 > W - 1 ? W - 1 : x0 + 1;
          float fy = iy - y0, fx = ix - x0;
          const float *p = img + (int64_t)c * H * W;
          v = (1 - fy) * (1 - fx) * p[(int64_t)y0 * W + x0] + (1 - fy) * fx * p[(int64_t)y0 * W + x1] +
              fy * (1 - fx) * p[(int64_t)y1 * W + x0] + fy * fx * p[(int64_t)y1 * W + x1];
        }
        out[(int64_t)c * H * W + (int64_t)y * W + x] = v;
      }
    }
}

/* ------------------------------------------------------------------------- */
/* a-6  preprocess.vgg.preprocess / deprocess                                 */
/* fast_artistic_video/preprocess.lua:48 (mean), :57-62, :66-71               */
/* ------------------------------------------------------------------------- */
static const float ORC_VGG_MEAN[3] = {103.939f, 116.779f, 123.68f}; /* preprocess.lua:48 */

/* in: 3xHxW RGB [0,1]; out[k] = in[2-k]*255 - mean[k]   (:61  index->mul->add(-1,mean)) */
ORC_API void orc_vgg_preprocess(const float *in, float *out, int64_t HW) {
  for (int k = 0; k < 3; ++k)
    for (int64_t i = 0; i < HW; ++i) out[k * HW + i] = in[(2 - k) * HW + i] * 255.0f - ORC_VGG_MEAN[k];
}

/* in: 3xHxW net output (BGR, mean-subtracted); out[2-k] = (in[k] + mean[k]) / 255   (:70) */
ORC_API void orc_vgg_deprocess(const float *in, float *out, int64_t HW) {
  for (int k = 0; k < 3; ++k)
    for (int64_t i = 0; i < HW; ++i) out[(2 - k) * HW + i] = (in[k * HW + i] + ORC_VGG_MEAN[k]) / 255.0f;
}

/* ------------------------------------------------------------------------- */
/* a-5  utils.min_filter(cert, r): 1 - maxpool_{r x r, s1, pad r/2}(1 - x)     */
/* fast_artistic_video/utils.lua:161-169                                      */
/* (-1*x)+1 -> maxpool (pad cells ignored) -> (-1*x)+1, all fp32               */
/* ------------------------------------------------------------------------- */
ORC_API void orc_min_filter(const float *in, float *out, int H, int W, int r) {
  int p = r / 2; /* math.floor(r/2), utils.lua:165 */
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float m = -INFINITY;
      /* SpatialMaxPooling window [y-p, y-p+r) clipped to the image */
      for (int dy = 0; dy < r; ++dy) {
        int yy = y - p + dy;
        if (yy < 0 || yy >= H) continue;
        for (int dx = 0; dx < r; ++dx) {
          int xx = x - p + dx;
          if (xx < 0 || xx >= W) continue;
          float t = in[(int64_t)yy * W + xx] * -1.0f + 1.0f;
          if (t > m) m = t;
        }
      }
      out[(int64_t)y * W + x] = m * -1.0f + 1.0f;
    }
}

/* ------------------------------------------------------------------------- */
/* a-8  run_next_image front half: 7-channel net input                        */
/* fast_artistic_video_core.lua:161-171, with fill_occlusions = 'vgg-mean'     */
/* (generate_fill :108-117 returns zeros) or an explicit fill tensor.          */
/*   in[0:3] = preprocess(content)                          (:168)             */
/*   in[3:6] = fill + cert * preprocess(warp(prev, flow))   (:166-167,:169)    */
/*   in[6]   = cert  (or min(cert, flow_mask))              (:169-170)         */
/* warp_mode: 0 = CUDA kernel semantics (a-1), 1 = image.warp pad semantics.   */
/* ------------------------------------------------------------------------- */
ORC_API void orc_temporal_input(const float *content, const float *prev, const float *flow,
                                const float *cert, const float *fill /* may be NULL */,
                                const float *flow_mask /* may be NULL */, float *out7, int H, int W,
                                int warp_mode) {
  int64_t HW = (int64_t)H * W;
  float *warped = (float *)malloc(sizeof(float) * 3 * HW);
  float *pre = (float *)malloc(sizeof(float) * 3 * HW);
  if (warp_mode == 0) {
    int64_t is[4] = {3 * HW, HW, W, 1}, gs[4] = {2 * HW, HW, W, 1};
    orc_warp_bdhw(prev, is, flow, gs, warped, is, 1, 3, H, W, H, W, 1);
  } else {
    orc_image_warp_pad(prev, flow, warped, 3, H, W, 0.0f);
  }
  orc_vgg_preprocess(warped, pre, HW); /* core.lua:166 */
  orc_vgg_preprocess(content, out7, HW); /* :168 */
  for (int k = 0; k < 3; ++k)
    for (int64_t i = 0; i < HW; ++i) {
      float masked = pre[k * HW + i] * cert[i];                        /* :167 cmul */
      out7[(3 + k) * HW + i] = (fill ? fill[k * HW + i] : 0.0f) + masked; /* :169 add */
    }
  for (int64_t i = 0; i < HW; ++i) {
    float m = cert[i];
    if (flow_mask && flow_mask[i] < m) m = flow_mask[i]; /* cmin :169 */
    out7[6 * HW + i] = m;
  }
  free(warped);
  free(pre);
}

/* a-9 run_image front half with model_img == nil (core.lua:133-137):          */
/* cat(pre(img), fill(cert=0) [zeros under vgg-mean], zeros(1ch))               */
ORC_API void orc_first_frame_input(const float *content, const float *fill, float *out7, int H,
                                   int W) {
  int64_t HW = (int64_t)H * W;
  orc_vgg_preprocess(content, out7, HW);
  for (int64_t i = 0; i < 3 * HW; ++i) out7[3 * HW + i] = fill ? fill[i] : 0.0f;
  for (int64_t i = 0; i < HW; ++i) out7[6 * HW + i] = 0.0f;
}

/* ------------------------------------------------------------------------- */
/* a-3 / a-13  Middlebury .flo                                                 */
/* flowFileLoader.lua:17-37 -> 2xHxW with [0]=v(dy), [1]=u(dx) (swap :31-32);  */
/* tag is read but not validated (:20).                                        */
/* consistencyChecker.cpp:16-36 -> planar (x,y,0)=u, (x,y,1)=v.                */
/* ------------------------------------------------------------------------- */
ORC_API int orc_flo_header(const char *path, int *W, int *H) {
  FILE *f = fopen(path, "rb");
  if (!f) return -1;
  float tag;
  int w, h;
  if (fread(&tag, 4, 1, f) != 1 || fread(&w, 4, 1, f) != 1 || fread(&h, 4, 1, f) != 1) {
    fclose(f);
    return -2;
  }
  fclose(f);
  *W = w;
  *H = h;
  return 0;
}

/* layout 0: Lua loader order (ch0 = v, ch1 = u); layout 1: checker order (ch0 = u, ch1 = v) */
ORC_API int orc_flo_read(const char *path, float *out, int layout) {
  FILE *f = fopen(path, "rb");
  if (!f) return -1;
  float tag;
  int W, H;
  if (fread(&tag, 4, 1, f) != 1 || fread(&W, 4, 1, f) != 1 || fread(&H, 4, 1, f) != 1) {
    fclose(f);
    return -2;
  }
  int64_t n = (int64_t)W * H;
  float *raw = (float *)malloc(sizeof(float) * 2 * n);
  if (fread(raw, sizeof(float), 2 * n, f) != (size_t)(2 * n)) {
    free(raw);
    fclose(f);
    return -3;
  }
  fclose(f);
  for (int64_t i = 0; i < n; ++i) {
    float u = raw[2 * i], v = raw[2 * i + 1];
    if (layout == 0) {
      out[i] = v;     /* flowFileLoader.lua:32 raw_flow[shift] = storage[2*shift+2] */
      out[n + i] = u; /* :31 */
    } else {
      out[i] = u; /* consistencyChecker.cpp:31 */
      out[n + i] = v; /* :32 */
    }
  }
  free(raw);
  return 0;
}

ORC_API int orc_flo_write(const char *path, const float *u, const float *v, int W, int H) {
  FILE *f = fopen(path, "wb");
  if (!f) return -1;
  float tag = 202021.25f; /* flowFileLoader.lua:11 "PIEH" */
  fwrite(&tag, 4, 1, f);
  fwrite(&W, 4, 1, f);
  fwrite(&H, 4, 1, f);
  for (int64_t i = 0; i < (int64_t)W * H; ++i) {
    fwrite(&u[i], 4, 1, f);
    fwrite(&v[i], 4, 1, f);
  }
  fclose(f);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* a-11 / a-12  consistencyChecker                                             */
/* ------------------------------------------------------------------------- */

/* NFilter::filter with CDerivative(3) = {-0.5, 0, 0.5}, mirrored borders.      */
/* CFilter.h:600-611 (taps), :1499-1533 (x), :1543-1578 (y).                    */
/* Accumulation order i = -1, 0, +1 starting from 0, all fp32.                  */
static void orc_deriv_x(const float *in, float *out, int W, int H) {
  const float f[3] = {-0.5f, 0.0f, 0.5f};
  int a2 = 2 * W - 1;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float s = 0;
      for (int i = -1; i < 2; ++i) {
        int xx = x + i;
        float v;
        if (xx < 0) v = in[(int64_t)y * W + (-1 - x - i)];
        else if (xx >= W) v = in[(int64_t)y * W + (a2 - x - i)];
        else v = in[(int64_t)y * W + xx];
        s += f[i + 1] * v;
      }
      out[(int64_t)y * W + x] = s;
    }
}
static void orc_deriv_y(const float *in, float *out, int W, int H) {
  const float f[3] = {-0.5f, 0.0f, 0.5f};
  int a2 = 2 * H - 1;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float s = 0;
      for (int i = -1; i < 2; ++i) {
        int yy = y + i;
        float v;
        if (yy < 0) v = in[(int64_t)(-1 - y - i) * W + x];
        else if (yy >= H) v = in[(int64_t)(a2 - y - i) * W + x];
        else v = in[(int64_t)yy * W + x];
        s += f[i + 1] * v;
      }
      out[(int64_t)y * W + x] = s;
    }
}

/* NFilter::recursiveSmoothX / Y, CFilter.h:1417-1439 / :1441-1464 */
typedef struct {
  float k, preMinus, prePlus, expSqr, twoExp;
} orc_iir_t;
static orc_iir_t orc_iir_coeffs(float sigma) {
  orc_iir_t c;
  float alpha = 2.5 / (sqrt(3.1415926535897932384626433832795) * sigma); /* NMath::Pi */
  float e = exp(-alpha);
  c.expSqr = e * e;
  c.twoExp = 2.0 * e;
  c.k = (1.0 - e) * (1.0 - e) / (1.0 + 2.0 * alpha * e - c.expSqr);
  c.preMinus = e * (alpha - 1.0);
  c.prePlus = e * (alpha + 1.0);
  return c;
}
static void orc_iir_line(const float *src, int64_t stride, int n, float *v1, float *v2, float *dst,
                         const orc_iir_t *c) {
#define S(i) src[(int64_t)(i) * stride]
  float k = c->k, pm = c->preMinus, pp = c->prePlus, e2 = c->expSqr, te = c->twoExp;
  v1[0] = (0.5f - k * pm) * S(0);
  v1[1] = k * (S(1) + pm * S(0)) + (te - e2) * v1[0];
  for (int x = 2; x < n; ++x) v1[x] = k * (S(x) + pm * S(x - 1)) + te * v1[x - 1] - e2 * v1[x - 2];
  v2[n - 1] = (0.5f + k * pm) * S(n - 1);
  v2[n - 2] = k * ((pp - e2) * S(n - 1)) + (te - e2) * v2[n - 1];
  for (int x = n - 3; x >= 0; --x)
    v2[x] = k * (pp * S(x + 1) - e2 * S(x + 2)) + te * v2[x + 1] - e2 * v2[x + 2];
  for (int x = 0; x < n; ++x) dst[(int64_t)x * stride] = v1[x] + v2[x];
#undef S
}
static void orc_recursive_smooth(float *m, int W, int H, float sigma) {
  orc_iir_t c = orc_iir_coeffs(sigma);
  int n = W > H ? W : H;
  float *v1 = (float *)malloc(sizeof(float) * n), *v2 = (float *)malloc(sizeof(float) * n);
  for (int y = 0; y < H; ++y) orc_iir_line(m + (int64_t)y * W, 1, W, v1, v2, m + (int64_t)y * W, &c);
  for (int x = 0; x < W; ++x) orc_iir_line(m + x, W, H, v1, v2, m + x, &c);
  free(v1);
  free(v2);
}

/*
 * computeCorners (consistencyChecker.cpp:39-78) followed by
 * structure.normalize(0,1) (CMatrix.h:721-736; called consistencyChecker.cpp:159).
 * image: Z planes of W x H (values 0..255 as read by CTensor::readFromPPM,
 * CTensor.h:888-936).  sqrt_mode 0: float temp - (float)sqrt; 1: double sqrt kept
 * in double until the subtraction result is rounded (see tests: pinned to _ref).
 */
ORC_API void orc_compute_corners(const float *image, int Z, int W, int H, float rho, float *corners,
                                 int do_normalize) {
  int64_t n = (int64_t)W * H;
  float *dx = (float *)malloc(sizeof(float) * n * Z), *dy = (float *)malloc(sizeof(float) * n * Z);
  for (int z = 0; z < Z; ++z) {
    orc_deriv_x(image + z * n, dx + z * n, W, H);
    orc_deriv_y(image + z * n, dy + z * n, W, H);
  }
  float *dxx = (float *)calloc(n, sizeof(float)), *dyy = (float *)calloc(n, sizeof(float)),
        *dxy = (float *)calloc(n, sizeof(float));
  for (int k = 0; k < Z; ++k) /* :55-61 */
    for (int64_t i = 0; i < n; ++i) {
      float gx = dx[k * n + i], gy = dy[k * n + i];
      dxx[i] += gx * gx;
      dyy[i] += gy * gy;
      dxy[i] += gx * gy;
    }
  orc_recursive_smooth(dxx, W, H, rho); /* :63-68 */
  orc_recursive_smooth(dyy, W, H, rho);
  orc_recursive_smooth(dxy, W, H, rho);
  for (int64_t i = 0; i < n; ++i) { /* :70-77 */
    float a = dxx[i], b = dxy[i], c = dyy[i];
    float temp = 0.5 * (a + c);
    float temp2 = temp * temp + b * b - a * c;
    if (temp2 < 0.0f) corners[i] = 0.0f;
    else corners[i] = temp - sqrt(temp2); /* C: double sqrt; the difference is formed in double */
  }
  if (do_normalize) { /* CMatrix.h:721-736 with aMin=0,aMax=1, initial min/max = +-30000 (:70) */
    float cmin = 30000, cmax = -30000;
    for (int64_t i = 0; i < n; ++i)
      if (corners[i] > cmax) cmax = corners[i];
      else if (corners[i] < cmin) cmin = corners[i];
    float t = cmax - cmin;
    if (t == 0) t = 1;
    else t = (1.0f - 0.0f) / t;
    for (int64_t i = 0; i < n; ++i) {
      corners[i] -= cmin;
      corners[i] *= t;
      corners[i] += 0.0f;
    }
  }
  free(dx); free(dy); free(dxx); free(dyy); free(dxy);
}

/* CMatrix::avg, CMatrix.h:1245-1251 */
ORC_API float orc_avg(const float *m, int64_t n) {
  float a = 0;
  for (int64_t i = 0; i < n; ++i) a += m[i];
  return a / (int)n;
}

/*
 * checkConsistency, consistencyChecker.cpp:80-134.
 * flow1/flow2: planar [2][H][W] with plane 0 = u (x-displacement), 1 = v.
 * structure: W x H or NULL (3-arg mode).  reliable: W x H, pre-set to 255 by the
 * caller (main :151).  Mixed float/double arithmetic mirrored exactly (:111-125).
 * The motion-edge branch (:129-132) writes MOTION_BOUNDARIE_VALUE = 255 (:12),
 * i.e. the value already there: kept for fidelity.
 */
ORC_API void orc_check_consistency(const float *flow1, const float *flow2, const float *structure,
                                   float *reliable, int W, int H) {
  int64_t size = (int64_t)W * H;
  float *fdx = (float *)malloc(sizeof(float) * 2 * size), *fdy = (float *)malloc(sizeof(float) * 2 * size);
  for (int z = 0; z < 2; ++z) {
    orc_deriv_x(flow1 + z * size, fdx + z * size, W, H);
    orc_deriv_y(flow1 + z * size, fdy + z * size, W, H);
  }
  float *motionEdge = (float *)calloc(size, sizeof(float));
  for (int64_t i = 0; i < size; ++i) { /* :88-93 */
    motionEdge[i] += fdx[i] * fdx[i];
    motionEdge[i] += fdx[size + i] * fdx[size + i];
    motionEdge[i] += fdy[i] * fdy[i];
    motionEdge[i] += fdy[size + i] * fdy[size + i];
  }
  float structureAvg = 0;
  if (structure) structureAvg = orc_avg(structure, size); /* :96-97 */
#define F1(x, y, z) flow1[(int64_t)W * ((int64_t)H * (z) + (y)) + (x)]
#define F2(x, y, z) flow2[(int64_t)W * ((int64_t)H * (z) + (y)) + (x)]
  for (int ay = 0; ay < H; ++ay)
    for (int ax = 0; ax < W; ++ax) {
      float bx = ax + F1(ax, ay, 0); /* :101 */
      float by = ay + F1(ax, ay, 1);
      int x1 = floor(bx); /* :103 */
      int y1 = floor(by);
      int x2 = x1 + 1;
      int y2 = y1 + 1;
      if (x1 < 0 || x2 >= W || y1 < 0 || y2 >= H) { /* :107-108 */
        reliable[(int64_t)ay * W + ax] = 0.0f;
        continue;
      }
      float alphaX = bx - x1;
      float alphaY = by - y1; /* :109 */
      float a = (1.0 - alphaX) * F2(x1, y1, 0) + alphaX * F2(x2, y1, 0); /* :110 */
      float b = (1.0 - alphaX) * F2(x1, y2, 0) + alphaX * F2(x2, y2, 0);
      float u = (1.0 - alphaY) * a + alphaY * b;
      a = (1.0 - alphaX) * F2(x1, y1, 1) + alphaX * F2(x2, y1, 1);
      b = (1.0 - alphaX) * F2(x1, y2, 1) + alphaX * F2(x2, y2, 1);
      float v = (1.0 - alphaY) * a + alphaY * b;
      float cx = bx + u; /* :116 */
      float cy = by + v;
      float u2 = F1(ax, ay, 0);
      float v2 = F1(ax, ay, 1);
      float structureTerm = 0;
      if (structure) { /* :122-123 */
        float s = structureAvg / 2.0f - structure[(int64_t)ay * W + ax];
        structureTerm = 4.0f / structureAvg * (0.0f > s ? 0.0f : s);
      }
      if (((cx - ax) * (cx - ax) + (cy - ay) * (cy - ay)) >=
          0.01 * (u2 * u2 + v2 * v2 + u * u + v * v) + structureTerm + 0.5f) { /* :124 */
        reliable[(int64_t)ay * W + ax] = 0.0f;
        continue;
      }
      if (motionEdge[(int64_t)ay * W + ax] > 0.01 * (u2 * u2 + v2 * v2) + 0.002f) { /* :128 */
        reliable[(int64_t)ay * W + ax] = 255; /* MOTION_BOUNDARIE_VALUE :12 */
        continue;
      }
    }
#undef F1
#undef F2
  free(fdx); free(fdy); free(motionEdge);
}

/* Whole-program restatement of main (consistencyChecker.cpp:136-172) on in-memory data. */
/* flows in checker layout (plane0=u).  image: 3 planes 0..255 or NULL.  out: u8 W*H.    */
ORC_API void orc_consistency_main(const float *flow1, const float *flow2, const float *image, int Z,
                                  int W, int H, uint8_t *out) {
  int64_t n = (int64_t)W * H;
  float *reliable = (float *)malloc(sizeof(float) * n);
  for (int64_t i = 0; i < n; ++i) reliable[i] = 255.0f; /* :150 */
  if (image) {
    float *structure = (float *)malloc(sizeof(float) * n);
    orc_compute_corners(image, Z, W, H, 3.0f, structure, 1); /* :157-158 */
    orc_check_consistency(flow1, flow2, structure, reliable, W, H);
    free(structure);
  } else {
    orc_check_consistency(flow1, flow2, NULL, reliable, W, H);
  }
  for (int64_t i = 0; i < n; ++i) { /* clip :169 + (char) cast in writeToPGM CMatrix.h:1068 */
    float r = reliable[i];
    if (r < 0.0f) r = 0.0f;
    else if (r > 255.0f) r = 255.0f;
    out[i] = (uint8_t)(int)r;
  }
  free(reliable);
}

/* binary PGM (P5) / PPM (P6) I/O --------------------------------------------- */
/* writer: CMatrix::writeToPGM, CMatrix.h:1059-1072 ("P5\n%d %d\n255\n")         */
ORC_API int orc_pgm_write(const char *path, const uint8_t *data, int W, int H) {
  FILE *f = fopen(path, "wb");
  if (!f) return -1;
  fprintf(f, "P5\n%d %d\n255\n", W, H);
  fwrite(data, 1, (size_t)W * H, f);
  fclose(f);
  return 0;
}
ORC_API int orc_ppm_write(const char *path, const uint8_t *rgb_interleaved, int W, int H) {
  FILE *f = fopen(path, "wb");
  if (!f) return -1;
  fprintf(f, "P6\n%d %d\n255\n", W, H);
  fwrite(rgb_interleaved, 1, (size_t)W * H * 3, f);
  fclose(f);
  return 0;
}

ORC_API int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
