// Render-quality metrics of re-rendered frames on the device (sm_90a): PSNR, MS-SSIM and the
// rendered-depth L1, batched over B frames.
//
// Replaces (reference @ f0366f20):
//   slam/common/common.py:429-479  save_render_imgs: np.clip, F.mse_loss / PSNR, the masked
//                                  depth L1 and pytorch_msssim.ms_ssim (data_range 1,
//                                  size_average) on the CPU, one frame per call
// Semantics (fixed here, documented in include/xrdslam_b200.h under xrd_eval_image_*): every fp32
// / fp64 operation is rounded to nearest in the order written (explicit intrinsics, no
// contraction), and every sum has a fixed order, so oracle/eval_image.py reproduces the results.
#include <cmath>

#include "common.cuh"

namespace xrd {
namespace evi {

constexpr int kLevels = XRD_EVAL_IMAGE_LEVELS;
constexpr int kWin = 11;
constexpr int kThreads = 256;
constexpr int kTileW = 32, kTileH = 16;                            // SSIM output tile
constexpr int kInW = kTileW + kWin - 1, kInH = kTileH + kWin - 1;  // the tile and its halo
constexpr int kChunk = kThreads * 16;                              // pixels per frame-sum block
constexpr float kC1 = (float)(0.01 * 0.01), kC2 = (float)(0.03 * 0.03);
__constant__ float kWeights[kLevels] = {0.0448f, 0.2856f, 0.3001f, 0.2363f, 0.1333f};

struct Win { float w[kWin]; };

// fp32 Gaussian, sigma 1.5, normalised by its in-order fp32 sum (host arithmetic is IEEE single)
Win gauss_window() {
  float g[kWin], s = 0.f;
  for (int k = 0; k < kWin; ++k) {
    const float d = (float)(k - kWin / 2);
    g[k] = (float)std::exp((double)(-(d * d) / 4.5f));
    s += g[k];
  }
  Win w;
  for (int k = 0; k < kWin; ++k) w.w[k] = g[k] / s;
  return w;
}

// One pyramid level of both images.  Level 0 reads the caller's HWC colours, clipping on load
// (and masking by gt depth > 0 when `mask` is set); levels 1..4 read planar [B][3][H][W] planes.
struct Level {
  const float* x;     // gt colour
  const float* y;     // rendered colour
  const float* mask;  // level 0 with XRD_EVAL_IMAGE_NO_DEPTH: gt depth [B][H][W], else null
  int H, W;
};

__device__ __forceinline__ float clip01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

template <bool kHwc>
__device__ __forceinline__ void load_pair(const Level& L, int b, int c, int yy, int xx, float& a,
                                          float& v) {
  if (kHwc) {
    const size_t px = ((size_t)b * L.H + yy) * L.W + xx;
    a = clip01(L.x[px * 3 + c]);
    v = clip01(L.y[px * 3 + c]);
    if (L.mask) {
      const float m = L.mask[px] > 0.f ? 1.f : 0.f;
      a = __fmul_rn(a, m);
      v = __fmul_rn(v, m);
    }
  } else {
    const size_t i = (((size_t)b * 3 + c) * L.H + yy) * L.W + xx;
    a = L.x[i];
    v = L.y[i];
  }
}

// fixed tree over the block's 256 values in red; -> the total, in every thread
__device__ __forceinline__ double tree_sum(double* red) {
  __syncthreads();
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// Per-frame sums, grid (chunks, B): thread t of chunk k takes pixels k * 4096 + t + 256 i.
// part [B][chunks][3] = (sum of squared colour errors, sum |gt - r| over gt > 0, count).
__global__ void __launch_bounds__(kThreads) k_frame_sums(const float* __restrict__ gt_color,
                                                         const float* __restrict__ color,
                                                         const float* __restrict__ gt_depth,
                                                         const double* __restrict__ depth,
                                                         int mask, int n_px,
                                                         double* __restrict__ part) {
  __shared__ double red[3][kThreads];
  const int k = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const size_t f = (size_t)b * n_px;
  double se = 0.0, dl = 0.0, dn = 0.0;
  for (int i = 0; i < kChunk / kThreads; ++i) {
    const int p = k * kChunk + i * kThreads + t;
    if (p >= n_px) break;
    const float g = gt_depth[f + p];
    const float m = g > 0.f ? 1.f : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float a = clip01(gt_color[(f + p) * 3 + c]), v = clip01(color[(f + p) * 3 + c]);
      if (mask) {
        a = __fmul_rn(a, m);
        v = __fmul_rn(v, m);
      }
      const float d = __fsub_rn(a, v);
      se = __dadd_rn(se, (double)__fmul_rn(d, d));
    }
    if (depth && g > 0.f) {
      dl = __dadd_rn(dl, fabs(__dsub_rn((double)g, depth[f + p])));
      dn = __dadd_rn(dn, 1.0);
    }
  }
  const double v[3] = {se, dl, dn};
  double* out = part + ((size_t)b * gridDim.x + k) * 3;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    red[j][t] = v[j];
    const double s = tree_sum(red[j]);
    if (t == 0) out[j] = s;
  }
}

// Level l -> planar level l + 1: avg_pool2d(2, 2, padding H % 2 / W % 2, count_include_pad), the
// 2x2 window summed row by row.
template <bool kHwc>
__global__ void __launch_bounds__(kThreads) k_pool(Level L, int Ho, int Wo, long long n,
                                                   float* __restrict__ ox,
                                                   float* __restrict__ oy) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const int xx = (int)(i % Wo), yy = (int)((i / Wo) % Ho);
  const int c = (int)((i / ((long long)Wo * Ho)) % 3), b = (int)(i / (3LL * Wo * Ho));
  const int r0 = 2 * yy - (L.H & 1), q0 = 2 * xx - (L.W & 1);
  float sa = 0.f, sv = 0.f;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int r = r0 + dy, q = q0 + dx;
      if (r < 0 || r >= L.H || q < 0 || q >= L.W) continue;  // zero padding
      float a, v;
      load_pair<kHwc>(L, b, c, r, q, a, v);
      sa = __fadd_rn(sa, a);
      sv = __fadd_rn(sv, v);
    }
  ox[i] = __fmul_rn(sa, 0.25f);
  oy[i] = __fmul_rn(sv, 0.25f);
}

// One level of SSIM, grid (tiles, 3 channels, B): stage a 32 x 16 output tile and its 10-pixel
// halo of both images, run the 11-tap pass along x then along y over the five maps, and write the
// tile's f64 sums of the ssim and cs maps to part [B][3][2][n_tiles].
template <bool kHwc>
__global__ void __launch_bounds__(kThreads) k_ssim(Level L, Win win, int tiles_x, int n_tiles,
                                                   double* __restrict__ part) {
  __shared__ float sx[kInH][kInW], sy[kInH][kInW];
  __shared__ float hs[5][kInH][kTileW];
  __shared__ double red[kThreads];
  const int tile = blockIdx.x, c = blockIdx.y, b = blockIdx.z, t = threadIdx.x;
  const int x0 = (tile % tiles_x) * kTileW, y0 = (tile / tiles_x) * kTileH;
  for (int i = t; i < kInH * kInW; i += kThreads) {
    const int r = i / kInW, q = i % kInW;
    float a = 0.f, v = 0.f;  // beyond the image: feeds only outputs outside the valid region
    if (y0 + r < L.H && x0 + q < L.W) load_pair<kHwc>(L, b, c, y0 + r, x0 + q, a, v);
    sx[r][q] = a;
    sy[r][q] = v;
  }
  __syncthreads();
  for (int i = t; i < kInH * kTileW; i += kThreads) {
    const int r = i / kTileW, q = i % kTileW;
    float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
      const float a = sx[r][q + k], v = sy[r][q + k], w = win.w[k];
      m[0] = __fadd_rn(m[0], __fmul_rn(w, a));
      m[1] = __fadd_rn(m[1], __fmul_rn(w, v));
      m[2] = __fadd_rn(m[2], __fmul_rn(w, __fmul_rn(a, a)));
      m[3] = __fadd_rn(m[3], __fmul_rn(w, __fmul_rn(v, v)));
      m[4] = __fadd_rn(m[4], __fmul_rn(w, __fmul_rn(a, v)));
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) hs[j][r][q] = m[j];
  }
  __syncthreads();
  const int q = t % kTileW, Ho = L.H - (kWin - 1), Wo = L.W - (kWin - 1);
  double s_ssim = 0.0, s_cs = 0.0;
  for (int r = t / kTileW; r < kTileH; r += kThreads / kTileW) {
    if (y0 + r >= Ho || x0 + q >= Wo) continue;
    float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < kWin; ++k)
#pragma unroll
      for (int j = 0; j < 5; ++j) m[j] = __fadd_rn(m[j], __fmul_rn(win.w[k], hs[j][r + k][q]));
    const float mu1_sq = __fmul_rn(m[0], m[0]), mu2_sq = __fmul_rn(m[1], m[1]);
    const float mu12 = __fmul_rn(m[0], m[1]);
    const float s1 = __fsub_rn(m[2], mu1_sq), s2 = __fsub_rn(m[3], mu2_sq);
    const float s12 = __fsub_rn(m[4], mu12);
    const float cs = __fdiv_rn(__fadd_rn(__fmul_rn(2.f, s12), kC2), __fadd_rn(__fadd_rn(s1, s2), kC2));
    const float l = __fdiv_rn(__fadd_rn(__fmul_rn(2.f, mu12), kC1),
                              __fadd_rn(__fadd_rn(mu1_sq, mu2_sq), kC1));
    s_ssim = __dadd_rn(s_ssim, (double)__fmul_rn(l, cs));
    s_cs = __dadd_rn(s_cs, (double)cs);
  }
  double* out = part + ((size_t)b * 3 + c) * 2 * n_tiles + tile;
  red[t] = s_ssim;
  const double a = tree_sum(red);
  red[t] = s_cs;
  const double d = tree_sum(red);
  if (t == 0) {
    out[0] = a;
    out[n_tiles] = d;
  }
}

struct Pyramid {
  int H[kLevels], W[kLevels], tiles_x[kLevels], n_tiles[kLevels];
  size_t part_off[kLevels];  // a level's first SSIM partial
  size_t n_part;
  int n_chunks;
};

Pyramid pyramid(int B, int H, int W) {
  Pyramid P;
  P.n_part = 0;
  for (int l = 0; l < kLevels; ++l) {
    P.H[l] = H;
    P.W[l] = W;
    P.tiles_x[l] = (W - (kWin - 1) + kTileW - 1) / kTileW;
    P.n_tiles[l] = P.tiles_x[l] * ((H - (kWin - 1) + kTileH - 1) / kTileH);
    P.part_off[l] = P.n_part;
    P.n_part += (size_t)B * 3 * 2 * P.n_tiles[l];
    H = (H + 1) / 2;
    W = (W + 1) / 2;
  }
  P.n_chunks = (int)((P.H[0] * (long long)P.W[0] + kChunk - 1) / kChunk);
  return P;
}

// finalize, one block per frame: ordered sums of the partials, then PSNR, depth L1 and MS-SSIM
__global__ void __launch_bounds__(kThreads) k_finalize(Pyramid P, int has_depth,
                                                       const double* __restrict__ frame_part,
                                                       const double* __restrict__ ssim_part,
                                                       double* __restrict__ out,
                                                       double* __restrict__ levels) {
  __shared__ double red[kThreads];
  __shared__ double mean[kLevels][3][2];
  const int b = blockIdx.x, t = threadIdx.x;
  double fs[3];
  for (int j = 0; j < 3; ++j) {
    const double* v = frame_part + (size_t)b * P.n_chunks * 3 + j;
    double s = 0.0;
    for (int i = t; i < P.n_chunks; i += kThreads) s = __dadd_rn(s, v[(size_t)i * 3]);
    red[t] = s;
    fs[j] = tree_sum(red);
  }
  for (int l = 0; l < kLevels; ++l) {
    const int n = P.n_tiles[l];
    const double cnt = (double)(P.H[l] - (kWin - 1)) * (double)(P.W[l] - (kWin - 1));
    for (int cj = 0; cj < 6; ++cj) {
      const double* v = ssim_part + P.part_off[l] + ((size_t)b * 6 + cj) * n;
      double s = 0.0;
      for (int i = t; i < n; i += kThreads) s = __dadd_rn(s, v[i]);
      red[t] = s;
      const double tot = tree_sum(red);
      if (t == 0) mean[l][cj / 2][cj % 2] = __ddiv_rn(tot, cnt);
    }
  }
  __syncthreads();
  if (t < kLevels * 6 && levels) levels[(size_t)b * kLevels * 6 + t] = (&mean[0][0][0])[t];
  if (t != 0) return;
  const double mse = __ddiv_rn(fs[0], 3.0 * (double)P.H[0] * (double)P.W[0]);
  double ch[3];
  for (int c = 0; c < 3; ++c) {
    double p = 1.0;
    for (int l = 0; l < kLevels; ++l) {
      const double v = mean[l][c][l == kLevels - 1 ? 0 : 1];
      const double r = v < 0.0 ? 0.0 : v;  // relu, NaN kept
      const double f = pow(r, (double)kWeights[l]);
      p = l == 0 ? f : __dmul_rn(p, f);
    }
    ch[c] = p;
  }
  double* o = out + (size_t)b * XRD_EVAL_IMAGE_OUT;
  o[0] = __dmul_rn(-10.0, log10(mse));
  o[1] = __ddiv_rn(__dadd_rn(__dadd_rn(ch[0], ch[1]), ch[2]), 3.0);
  o[2] = has_depth ? __dmul_rn(__ddiv_rn(fs[1], fs[2]), 100.0) : 0.0;
  o[3] = mse;
}

struct ImageWs : Carver {
  ImageWs(void* base, int B, const Pyramid& P)
      : Carver(base), frame_part(take<double>((size_t)B * P.n_chunks * 3)),
        ssim_part(take<double>(P.n_part)) {
    x[0] = y[0] = nullptr;
    for (int l = 1; l < kLevels; ++l) {
      const size_t n = (size_t)B * 3 * P.H[l] * P.W[l];
      x[l] = take<float>(n);
      y[l] = take<float>(n);
    }
  }
  double* frame_part;
  double* ssim_part;
  float* x[kLevels];
  float* y[kLevels];
};

bool shape_ok(int B, int H, int W, int flags) {
  return B >= 1 && B <= 65535 && H >= XRD_EVAL_IMAGE_MIN_SIDE && W >= XRD_EVAL_IMAGE_MIN_SIDE &&
         H <= XRD_EVAL_IMAGE_MAX_SIDE && W <= XRD_EVAL_IMAGE_MAX_SIDE &&
         (flags & ~XRD_EVAL_IMAGE_NO_DEPTH) == 0;
}

}  // namespace evi
}  // namespace xrd

using namespace xrd;
using namespace xrd::evi;

extern "C" size_t xrd_eval_image_workspace_bytes(int B, int H, int W) {
  if (!shape_ok(B, H, W, 0)) return 0;
  return ImageWs(nullptr, B, pyramid(B, H, W)).bytes();
}

extern "C" int xrd_eval_image_metrics(const float* gt_color, const float* color,
                                      const float* gt_depth, const double* depth, int B, int H,
                                      int W, int flags, double* out, double* levels,
                                      void* workspace, size_t workspace_bytes, void* stream_) {
  if (!shape_ok(B, H, W, flags)) return XRD_E_SHAPE;
  const bool has_depth = !(flags & XRD_EVAL_IMAGE_NO_DEPTH);
  if (!gt_color || !color || !gt_depth || (has_depth && !depth) || !out || !workspace)
    return XRD_E_NULL;
  const Pyramid P = pyramid(B, H, W);
  const ImageWs L(workspace, B, P);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t s = (cudaStream_t)stream_;
  static const Win win = gauss_window();
  {
    KernelTimer timer(s);
    k_frame_sums<<<dim3(P.n_chunks, B), kThreads, 0, s>>>(gt_color, color, gt_depth,
                                                           has_depth ? depth : nullptr,
                                                           !has_depth, H * W, L.frame_part);
    XRD_LAUNCH_CHECK();
    for (int l = 0; l < kLevels; ++l) {
      const Level lv = l == 0 ? Level{gt_color, color, has_depth ? nullptr : gt_depth, H, W}
                              : Level{L.x[l], L.y[l], nullptr, P.H[l], P.W[l]};
      const dim3 grid(P.n_tiles[l], 3, B);
      double* part = L.ssim_part + P.part_off[l];
      if (l == 0)
        k_ssim<true><<<grid, kThreads, 0, s>>>(lv, win, P.tiles_x[l], P.n_tiles[l], part);
      else
        k_ssim<false><<<grid, kThreads, 0, s>>>(lv, win, P.tiles_x[l], P.n_tiles[l], part);
      XRD_LAUNCH_CHECK();
      if (l + 1 == kLevels) break;
      const long long n = 3LL * B * P.H[l + 1] * P.W[l + 1];
      if (l == 0)
        k_pool<true><<<blocks(n, kThreads), kThreads, 0, s>>>(lv, P.H[1], P.W[1], n, L.x[1], L.y[1]);
      else
        k_pool<false><<<blocks(n, kThreads), kThreads, 0, s>>>(lv, P.H[l + 1], P.W[l + 1], n,
                                                               L.x[l + 1], L.y[l + 1]);
      XRD_LAUNCH_CHECK();
    }
    k_finalize<<<B, kThreads, 0, s>>>(P, has_depth, L.frame_part, L.ssim_part, out, levels);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}
