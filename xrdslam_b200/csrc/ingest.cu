// Frame ingest (sm_90a): decoded uint8 BGR colour and uint16 (PNG) or float32 (EXR) depth -> the
// float32 frames the reference's BaseDataset.__getitem__ (slam/common/datasets.py:95-134)
// produces, stage by stage in the same arithmetic:
//   undistort (colour, uint8; cv::undistort's map and fixed-point remap) -> BGR->RGB, / 255. in
//   f64 -> depth f32(d) / f32(scale) -> colour resized to the depth's size (cv2.resize
//   INTER_LINEAR on f64) -> crop -> downsample (colour INTER_LINEAR, depth INTER_NEAREST) -> f32.
// Every floating-point operation is an explicit round-to-nearest intrinsic, so nothing is
// contracted into an FMA: cv2's own C++ code has none.  oracle/ingest.py restates this file.
#include <float.h>

#include <algorithm>

#include "common.cuh"

namespace xrd {
namespace ingest {

constexpr int kThreads = 256;
constexpr int kInterBits = 5, kInterTab = 1 << kInterBits;  // map fractions: 1/32 pixel
constexpr int kCoefBits = 15;                                // remap weights: 2^15 fixed point
constexpr int kStripePixels = 1 << 12;                       // cv::undistort's stripe: 4096 / W rows
constexpr int kMaxSide = 32767;                              // CV_16SC2 map range

enum Mode : int { kCopy = 0, kLinear = 1, kArea2 = 2 };

// One resize of cv::resize: src (sh, sw) -> dst (dh, dw).  scale = 1 / (dst / src) per axis.
struct Resize {
  int mode, sh, sw;
  double scale_x, scale_y;
};

struct Params {
  int B, H0, W0, Hd, Wd, h, w, edge, hc, wc;
  Resize r1, r2;  // colour -> depth size; cropped -> output (mode kCopy when f == 1)
  double nn_scale_x, nn_scale_y;
  float depth_scale;
};

struct Distortion {
  double fx, fy, cx, cy;
  double k[12];  // k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4
  int stripe;
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// cv::undistort of one pixel (x, y) of frame b, all three channels.
// initUndistortRectifyMap (new camera matrix = K, R = I) in the row stripe of y: the inverse of
// the stripe's camera matrix by cv::invert's 3x3 cofactor formula, the distortion model, then
// CV_16SC2 + CV_16UC1 maps (cvRound(u * 32)); remap INTER_LINEAR on uint8 with 15-bit weights and
// BORDER_CONSTANT 0.
__global__ void __launch_bounds__(kThreads)
k_undistort(const uint8_t* __restrict__ src, Distortion D, int B, int H, int W,
            uint8_t* __restrict__ dst) {
  const long long n = (long long)B * H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int x = (int)(p % W);
  const int y = (int)((p / W) % H);
  const int b = (int)(p / ((long long)W * H));
  const int y0 = y / D.stripe * D.stripe;
  const double fx = D.fx, fy = D.fy, cx = D.cx, cy = D.cy;
  const double cyp = dsub(cy, (double)y0);
  const double d = ddiv(1.0, dmul(fx, fy));
  const double ir0 = dmul(fy, d);
  const double ir2 = dmul(dsub(0.0, dmul(cx, fy)), d);
  const double ir4 = dmul(fx, d);
  const double ir5 = dmul(dsub(0.0, dmul(fx, cyp)), d);
  const double ir8 = dmul(dmul(fx, fy), d);
  const double _x = dadd(ir2, dmul((double)x, ir0));
  const double _y = dadd(dmul((double)(y - y0), ir4), ir5);
  const double iw = ddiv(1.0, ir8);
  const double xx = dmul(_x, iw), yy = dmul(_y, iw);
  const double x2 = dmul(xx, xx), y2 = dmul(yy, yy);
  const double r2 = dadd(x2, y2);
  const double xy2 = dmul(dmul(2.0, xx), yy);
  const double* k = D.k;
  const double num = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k[4], r2), k[1]), r2), k[0]), r2));
  const double den = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k[7], r2), k[6]), r2), k[5]), r2));
  const double kr = ddiv(num, den);
  const double xd = dadd(dadd(dadd(dadd(dmul(xx, kr), dmul(k[2], xy2)),
                                   dmul(k[3], dadd(r2, dmul(2.0, x2)))),
                              dmul(k[8], r2)),
                         dmul(dmul(k[9], r2), r2));
  const double yd = dadd(dadd(dadd(dadd(dmul(yy, kr), dmul(k[2], dadd(r2, dmul(2.0, y2)))),
                                   dmul(k[3], xy2)),
                              dmul(k[10], r2)),
                         dmul(dmul(k[11], r2), r2));
  const double u = dadd(dmul(fx, xd), cx);
  const double v = dadd(dmul(fy, yd), cy);
  const long long iu = __double2ll_rn(dmul(u, (double)kInterTab));
  const long long iv = __double2ll_rn(dmul(v, (double)kInterTab));
  const int sx = (int)(iu >> kInterBits), sy = (int)(iv >> kInterBits);
  const int ax = (int)(iu & (kInterTab - 1)), ay = (int)(iv & (kInterTab - 1));
  const int wt[4] = {(kInterTab - ax) * (kInterTab - ay) * kInterTab,
                     ax * (kInterTab - ay) * kInterTab, (kInterTab - ax) * ay * kInterTab,
                     ax * ay * kInterTab};
  int acc[3] = {0, 0, 0};
  const uint8_t* img = src + (long long)b * H * W * 3;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int cx_ = sx + (c & 1), cy_ = sy + (c >> 1);
    if (cx_ < 0 || cx_ >= W || cy_ < 0 || cy_ >= H) continue;
    const uint8_t* s = img + ((long long)cy_ * W + cx_) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) acc[ch] += (int)s[ch] * wt[c];
  }
  uint8_t* o = dst + p * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) o[ch] = (uint8_t)min((acc[ch] + (1 << (kCoefBits - 1))) >> kCoefBits, 255);
}

// cv::resize INTER_LINEAR's index and float32 weight of destination index d: t = float((d + 0.5)
// * scale - 0.5), s = floor(t), t -= s.  Along x an index below 0 or at/after src - 1 is clamped
// with weight (1, 0); along y the rows are clamped when fetched.
struct Tap {
  int s0, s1;
  double a0, a1;
};

__device__ __forceinline__ Tap linear_tap(int d, double scale, int src, bool clamp) {
  float t = __double2float_rn(dsub(dmul(dadd((double)d, 0.5), scale), 0.5));
  int s = (int)floorf(t);
  t = __fsub_rn(t, (float)s);
  if (clamp) {
    if (s < 0) t = 0.f, s = 0;
    if (s >= src - 1) t = 0.f, s = src - 1;
  }
  Tap tp;
  tp.s0 = min(max(s, 0), src - 1);
  tp.s1 = min(max(s + 1, 0), src - 1);
  tp.a0 = (double)__fsub_rn(1.f, t);
  tp.a1 = (double)t;
  return tp;
}

// Colour after the BGR->RGB swap and / 255.: channel ch (RGB) of source pixel (y, x).
struct Source {
  const uint8_t* img;
  int W;
  __device__ __forceinline__ double operator()(int y, int x, int ch) const {
    return ddiv((double)img[((long long)y * W + x) * 3 + (2 - ch)], 255.0);
  }
};

// Stage 1 (resize to the depth's size), read through the crop offset.
struct Stage1 {
  Source src;
  Resize r;
  int edge;
  __device__ __forceinline__ double operator()(int y, int x, int ch) const {
    y += edge;
    x += edge;
    return sample(src, r, y, x, ch);
  }
  template <class S>
  __device__ static double sample(const S& f, const Resize& r, int y, int x, int ch) {
    if (r.mode == kCopy) return f(y, x, ch);
    if (r.mode == kArea2) {
      // cv::resize's fast area path: (((0 + s00) + s01) + s10) + s11, times 0.25f
      const int y0 = 2 * y, x0 = 2 * x;
      double sum = dadd(0.0, f(y0, x0, ch));
      sum = dadd(sum, f(y0, x0 + 1, ch));
      sum = dadd(sum, f(y0 + 1, x0, ch));
      sum = dadd(sum, f(y0 + 1, x0 + 1, ch));
      return dmul(sum, 0.25);
    }
    const Tap tx = linear_tap(x, r.scale_x, r.sw, true);
    const Tap ty = linear_tap(y, r.scale_y, r.sh, false);
    const double h0 = dadd(dmul(f(ty.s0, tx.s0, ch), tx.a0), dmul(f(ty.s0, tx.s1, ch), tx.a1));
    const double h1 = dadd(dmul(f(ty.s1, tx.s0, ch), tx.a0), dmul(f(ty.s1, tx.s1, ch), tx.a1));
    return dadd(dmul(h0, ty.a0), dmul(h1, ty.a1));
  }
};

// Stage 3 on one depth value: f32(d) / f32(png_depth_scale).  uint16 depth converts exactly.
__device__ __forceinline__ float depth_div(uint16_t d, float scale) {
  return __fdiv_rn((float)d, scale);
}

// float32 depth as numpy divides it on x86 (SSE divss): a NaN operand comes back quietened with
// its payload (the dividend's first), and an invalid division (inf / inf, 0 / 0) gives x86's
// default NaN 0xffc00000, where the device's division would return 0x7fffffff in both cases.
// Infinities, signed zeros and subnormals follow IEEE division, as __fdiv_rn does.
__device__ __forceinline__ float depth_div(float d, float scale) {
  constexpr unsigned kQuiet = 0x00400000u, kDefaultNaN = 0xffc00000u;
  if (isnan(d)) return __uint_as_float(__float_as_uint(d) | kQuiet);
  if (isnan(scale)) return __uint_as_float(__float_as_uint(scale) | kQuiet);
  const float q = __fdiv_rn(d, scale);
  return isnan(q) ? __uint_as_float(kDefaultNaN) : q;
}

// One thread per output pixel: colour (3 channels) and depth.  DepthT is uint16_t (PNG depth) or
// float (EXR depth); only stage 3 reads it.
template <class DepthT>
__global__ void __launch_bounds__(kThreads)
k_ingest(const uint8_t* __restrict__ color, const DepthT* __restrict__ depth, Params P,
         float* __restrict__ rgb, float* __restrict__ depth_out) {
  const long long n = (long long)P.B * P.h * P.w;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int x = (int)(p % P.w);
  const int y = (int)((p / P.w) % P.h);
  const int b = (int)(p / ((long long)P.w * P.h));
  const Stage1 s1{Source{color + (long long)b * P.H0 * P.W0 * 3, P.W0}, P.r1, P.edge};
#pragma unroll 1
  for (int ch = 0; ch < 3; ++ch)
    rgb[p * 3 + ch] = __double2float_rn(Stage1::sample(s1, P.r2, y, x, ch));
  int dy = y, dx = x;
  if (P.r2.mode != kCopy) {
    dx = min((int)floor(dmul((double)x, P.nn_scale_x)), P.wc - 1);
    dy = min((int)floor(dmul((double)y, P.nn_scale_y)), P.hc - 1);
  }
  const DepthT dv = depth[((long long)b * P.Hd + dy + P.edge) * P.Wd + dx + P.edge];
  depth_out[p] = depth_div(dv, P.depth_scale);
}

// cv::resize's scale per axis and its choice of path
Resize make_resize(int sh, int sw, int dh, int dw) {
  Resize r{kCopy, sh, sw, 1.0, 1.0};
  if (sh == dh && sw == dw) return r;
  r.scale_x = 1.0 / ((double)dw / (double)sw);
  r.scale_y = 1.0 / ((double)dh / (double)sh);
  const bool area2 = fabs(r.scale_x - 2.0) < DBL_EPSILON && fabs(r.scale_y - 2.0) < DBL_EPSILON;
  r.mode = area2 ? kArea2 : kLinear;
  return r;
}

bool params(const XrdIngestCfg* c, Params* P) {
  if (c->B < 1 || c->B > 65535 || c->H0 < 1 || c->W0 < 1 || c->Hd < 1 || c->Wd < 1 ||
      c->H0 > kMaxSide || c->W0 > kMaxSide || c->Hd > kMaxSide || c->Wd > kMaxSide)
    return false;
  if (!(c->n_dist == 0 || c->n_dist == 4 || c->n_dist == 5 || c->n_dist == 8 || c->n_dist == 12))
    return false;
  if (c->crop_edge < 0 || c->downsample_factor < 1 || !(c->png_depth_scale != 0.0)) return false;
  const int f = c->downsample_factor;
  P->B = c->B, P->H0 = c->H0, P->W0 = c->W0, P->Hd = c->Hd, P->Wd = c->Wd;
  P->edge = c->crop_edge;
  P->hc = c->Hd - 2 * c->crop_edge;
  P->wc = c->Wd - 2 * c->crop_edge;
  P->h = f > 1 ? P->hc / f : P->hc;
  P->w = f > 1 ? P->wc / f : P->wc;
  if (P->hc < 1 || P->wc < 1 || P->h < 1 || P->w < 1) return false;
  P->r1 = make_resize(c->H0, c->W0, c->Hd, c->Wd);
  P->r2 = f > 1 ? make_resize(P->hc, P->wc, P->h, P->w) : make_resize(1, 1, 1, 1);
  P->nn_scale_x = 1.0 / ((double)P->w / (double)P->wc);
  P->nn_scale_y = 1.0 / ((double)P->h / (double)P->hc);
  P->depth_scale = (float)c->png_depth_scale;
  return true;
}

// the undistorted colour frames, when there is a distortion model
struct IngestWs : Carver {
  IngestWs(void* base, const XrdIngestCfg& c)
      : Carver(base),
        undistorted(take<uint8_t>(c.n_dist ? (size_t)c.B * c.H0 * c.W0 * 3 : 0)) {}
  uint8_t* undistorted;
};

}  // namespace ingest
}  // namespace xrd

using namespace xrd;
using namespace xrd::ingest;

extern "C" size_t xrd_frame_ingest_workspace_bytes(const XrdIngestCfg* cfg) {
  Params P;
  if (!cfg || !params(cfg, &P)) return 0;
  return IngestWs(nullptr, *cfg).bytes();
}

namespace {

template <class DepthT>
int frame_ingest(const XrdIngestCfg* cfg, const uint8_t* color, const DepthT* depth, float* rgb,
                 float* depth_out, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!cfg) return XRD_E_NULL;
  Params P;
  if (!params(cfg, &P)) return XRD_E_SHAPE;
  if (!color || !depth || !rgb || !depth_out) return XRD_E_NULL;
  const IngestWs L(workspace, *cfg);
  if (L.bytes() > 0 && !workspace) return XRD_E_NULL;
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t s = (cudaStream_t)stream_;
  KernelTimer timer(s);
  const uint8_t* src = color;
  if (cfg->n_dist) {
    Distortion D;
    D.fx = cfg->fx, D.fy = cfg->fy, D.cx = cfg->cx, D.cy = cfg->cy;
    for (int i = 0; i < 12; ++i) D.k[i] = i < cfg->n_dist ? cfg->dist[i] : 0.0;
    D.stripe = std::min(std::max(1, kStripePixels / cfg->W0), cfg->H0);
    const long long n = (long long)cfg->B * cfg->H0 * cfg->W0;
    k_undistort<<<blocks(n, kThreads), kThreads, 0, s>>>(color, D, cfg->B, cfg->H0, cfg->W0,
                                                         L.undistorted);
    XRD_LAUNCH_CHECK();
    src = L.undistorted;
  }
  const long long n = (long long)P.B * P.h * P.w;
  k_ingest<DepthT><<<blocks(n, kThreads), kThreads, 0, s>>>(src, depth, P, rgb, depth_out);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

}  // namespace

extern "C" int xrd_frame_ingest(const XrdIngestCfg* cfg, const uint8_t* color,
                                const uint16_t* depth, float* rgb, float* depth_out,
                                void* workspace, size_t workspace_bytes, void* stream) {
  return frame_ingest(cfg, color, depth, rgb, depth_out, workspace, workspace_bytes, stream);
}

extern "C" int xrd_frame_ingest_f32(const XrdIngestCfg* cfg, const uint8_t* color,
                                    const float* depth, float* rgb, float* depth_out,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  return frame_ingest(cfg, color, depth, rgb, depth_out, workspace, workspace_bytes, stream);
}
