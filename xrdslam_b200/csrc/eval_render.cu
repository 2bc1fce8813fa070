// ds-eval's 2D depth-L1 metric on the device (sm_90a): a batched mesh depth rasteriser, the
// unseen-region check of candidate views and the per-view |gt - rec| sums.
//
// Replaces (reference @ f0366f20):
//   scripts/utils/eval_recon.py:66-90    check_proj (torch, one candidate view per call)
//   scripts/utils/eval_recon.py:234-278  open3d Visualizer depth captures of both meshes and the
//                                        per-view mean of |gt - rec| over rec > 0 (numpy f32)
// Semantics (fixed here, documented in include/xrdslam_b200.h under xrd_eval_render_* /
// xrd_eval_points_seen / xrd_eval_depth_l1): every fp32 / fp64 operation is rounded to nearest in
// the order written (explicit intrinsics, no contraction); coverage is decided by exact int64
// edge functions on a 1/256-pixel grid; the depth buffer is a min over fragments, so the image
// does not depend on the order in which triangles are drawn.
#include <cmath>

#include "common.cuh"

namespace xrd {
namespace evr {

constexpr int kSub = XRD_EVAL_RENDER_SUBPIXEL;   // fixed-point steps per pixel (2^8)
constexpr int kSubShift = 8;
constexpr int kInline = XRD_EVAL_RENDER_INLINE_PX;  // largest pixel box rasterised inline
constexpr int kMaxViews = XRD_EVAL_RENDER_MAX_VIEWS;
constexpr double kGuard = XRD_EVAL_RENDER_GUARD;    // |u - cx|, |v - cy| bound in pixels
constexpr int kMaxPoly = 8;                          // triangle clipped by 5 planes

struct Cam {
  int H, W;
  double fx, fy, cx, cy, near, far;
};

struct V3 { double x, y, z; };

// camera-space point ((r0 x + r1 y) + r2 z) + t per row
__device__ __forceinline__ V3 to_cam(const double* __restrict__ M, double x, double y, double z) {
  V3 p;
  p.x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[0], x), __dmul_rn(M[1], y)), __dmul_rn(M[2], z)), M[3]);
  p.y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[4], x), __dmul_rn(M[5], y)), __dmul_rn(M[6], z)), M[7]);
  p.z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[8], x), __dmul_rn(M[9], y)), __dmul_rn(M[10], z)), M[11]);
  return p;
}

// signed distance to clip plane k (inside >= 0): 0 near, 1 u <= cx + G, 2 u >= cx - G,
// 3 v <= cy + G, 4 v >= cy - G (planes through the camera centre; z > 0 after plane 0)
__device__ __forceinline__ double plane_d(const Cam& c, int k, const V3& p) {
  switch (k) {
    case 0: return __dsub_rn(p.z, c.near);
    case 1: return __dsub_rn(__dmul_rn(kGuard, p.z), __dmul_rn(c.fx, p.x));
    case 2: return __dadd_rn(__dmul_rn(kGuard, p.z), __dmul_rn(c.fx, p.x));
    case 3: return __dsub_rn(__dmul_rn(kGuard, p.z), __dmul_rn(c.fy, p.y));
    default: return __dadd_rn(__dmul_rn(kGuard, p.z), __dmul_rn(c.fy, p.y));
  }
}

__device__ __forceinline__ bool inside_all(const Cam& c, const V3& p) {
#pragma unroll
  for (int k = 0; k < 5; ++k)
    if (plane_d(c, k, p) < 0.0) return false;
  return true;
}

__device__ __forceinline__ bool less_xyz(const V3& a, const V3& b) {
  return a.x < b.x || (a.x == b.x && (a.y < b.y || (a.y == b.y && a.z < b.z)));
}

// point where segment (a, b) crosses plane k, computed from the lexicographically smaller end
// so that two triangles sharing the segment get the same point
__device__ __forceinline__ V3 cross_point(const Cam& c, int k, V3 a, V3 b) {
  if (less_xyz(b, a)) { const V3 t = a; a = b; b = t; }
  const double da = plane_d(c, k, a), db = plane_d(c, k, b);
  const double t = __ddiv_rn(da, __dsub_rn(da, db));
  return V3{__dadd_rn(a.x, __dmul_rn(t, __dsub_rn(b.x, a.x))),
            __dadd_rn(a.y, __dmul_rn(t, __dsub_rn(b.y, a.y))),
            __dadd_rn(a.z, __dmul_rn(t, __dsub_rn(b.z, a.z)))};
}

// Sutherland-Hodgman against planes 0..4 in order; -> vertex count (0 or 3..8) in P
__device__ int clip_poly(const Cam& c, V3 (&P)[kMaxPoly + 1], int n) {
  V3 Q[kMaxPoly + 1];
  for (int k = 0; k < 5 && n > 0; ++k) {
    int m = 0;
    for (int i = 0; i < n; ++i) {
      const V3 cur = P[i], prev = P[i == 0 ? n - 1 : i - 1];
      const bool ci = plane_d(c, k, cur) >= 0.0, pi = plane_d(c, k, prev) >= 0.0;
      if (ci) {
        if (!pi) Q[m++] = cross_point(c, k, prev, cur);
        Q[m++] = cur;
      } else if (pi) {
        Q[m++] = cross_point(c, k, prev, cur);
      }
    }
    n = m < 3 ? 0 : min(m, kMaxPoly);
    for (int i = 0; i < n; ++i) P[i] = Q[i];
  }
  return n;
}

// 1/z over the image is affine for a plane: 1/z = (ax i + ay j) + c0 with the plane n.p = k of
// the unclipped triangle (n = e1 x e2 in camera space).  -> false when the plane passes
// through the camera centre (k == 0).
struct Plane { double ax, ay, c0, k; };

__device__ __forceinline__ bool tri_plane(const Cam& c, const V3& p0, const V3& p1, const V3& p2,
                                          Plane& pl) {
  const double e1x = __dsub_rn(p1.x, p0.x), e1y = __dsub_rn(p1.y, p0.y), e1z = __dsub_rn(p1.z, p0.z);
  const double e2x = __dsub_rn(p2.x, p0.x), e2y = __dsub_rn(p2.y, p0.y), e2z = __dsub_rn(p2.z, p0.z);
  const double nx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double ny = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double nz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  pl.k = __dadd_rn(__dadd_rn(__dmul_rn(nx, p0.x), __dmul_rn(ny, p0.y)), __dmul_rn(nz, p0.z));
  pl.ax = __ddiv_rn(nx, c.fx);
  pl.ay = __ddiv_rn(ny, c.fy);
  pl.c0 = __dsub_rn(nz, __dadd_rn(__dmul_rn(pl.ax, c.cx), __dmul_rn(pl.ay, c.cy)));
  return pl.k != 0.0;
}

// fragment depth at pixel (i, j): fp32(k / ((ax i + ay j) + c0)); 0 when dropped (not in
// (0, far] or not finite)
__device__ __forceinline__ float frag_depth(const Cam& c, const Plane& pl, int i, int j) {
  const double den = __dadd_rn(__dadd_rn(__dmul_rn(pl.ax, (double)i), __dmul_rn(pl.ay, (double)j)), pl.c0);
  const float z = __double2float_rn(__ddiv_rn(pl.k, den));
  return (z > 0.f && z <= (float)c.far && isfinite(z)) ? z : 0.f;
}

struct Snapped {
  long long X[3], Y[3], area;
  int x0, x1, y0, y1;  // inclusive pixel box, clamped to the image
};

__device__ __forceinline__ long long snap(double v) { return __double2ll_rn(__dmul_rn(v, (double)kSub)); }

__device__ __forceinline__ void project(const Cam& c, const V3& p, long long& X, long long& Y) {
  X = snap(__dadd_rn(__ddiv_rn(__dmul_rn(c.fx, p.x), p.z), c.cx));
  Y = snap(__dadd_rn(__ddiv_rn(__dmul_rn(c.fy, p.y), p.z), c.cy));
}

// -> false when the triangle covers no pixel centre box or has zero area
__device__ __forceinline__ bool setup(const Cam& c, const V3& a, const V3& b, const V3& d, Snapped& s) {
  project(c, a, s.X[0], s.Y[0]);
  project(c, b, s.X[1], s.Y[1]);
  project(c, d, s.X[2], s.Y[2]);
  const long long xmn = min(s.X[0], min(s.X[1], s.X[2])), xmx = max(s.X[0], max(s.X[1], s.X[2]));
  const long long ymn = min(s.Y[0], min(s.Y[1], s.Y[2])), ymx = max(s.Y[0], max(s.Y[1], s.Y[2]));
  s.x0 = (int)max(0LL, (xmn + kSub - 1) >> kSubShift);
  s.x1 = (int)min((long long)c.W - 1, xmx >> kSubShift);
  s.y0 = (int)max(0LL, (ymn + kSub - 1) >> kSubShift);
  s.y1 = (int)min((long long)c.H - 1, ymx >> kSubShift);
  if (s.x0 > s.x1 || s.y0 > s.y1) return false;
  s.area = (s.X[1] - s.X[0]) * (s.Y[2] - s.Y[0]) - (s.Y[1] - s.Y[0]) * (s.X[2] - s.X[0]);
  return s.area != 0;
}

// inclusive coverage: every edge function has the area's sign or is zero
__device__ __forceinline__ bool covers(const Snapped& s, int i, int j) {
  const long long px = (long long)i << kSubShift, py = (long long)j << kSubShift;
  const long long w0 = (s.X[2] - s.X[1]) * (py - s.Y[1]) - (s.Y[2] - s.Y[1]) * (px - s.X[1]);
  const long long w1 = (s.X[0] - s.X[2]) * (py - s.Y[2]) - (s.Y[0] - s.Y[2]) * (px - s.X[2]);
  const long long w2 = (s.X[1] - s.X[0]) * (py - s.Y[0]) - (s.Y[1] - s.Y[0]) * (px - s.X[0]);
  return s.area > 0 ? (w0 >= 0 && w1 >= 0 && w2 >= 0) : (w0 <= 0 && w1 <= 0 && w2 <= 0);
}

// depth min through the complemented bits of a positive float: the max of ~bits is the min
// depth, and 0 stays "nothing drawn"
__device__ __forceinline__ void write_depth(unsigned* img, int W, int i, int j, float z) {
  if (z > 0.f) atomicMax(img + (size_t)j * W + i, ~__float_as_uint(z));
}

__device__ __forceinline__ bool load_face(const float* __restrict__ V, int nV,
                                          const int32_t* __restrict__ F, int f, V3 (&w)[3]) {
  const int i0 = F[3 * f], i1 = F[3 * f + 1], i2 = F[3 * f + 2];
  if (i0 < 0 || i0 >= nV || i1 < 0 || i1 >= nV || i2 < 0 || i2 >= nV) return false;
  const int id[3] = {i0, i1, i2};
#pragma unroll
  for (int k = 0; k < 3; ++k)
    w[k] = V3{(double)V[3 * id[k]], (double)V[3 * id[k] + 1], (double)V[3 * id[k] + 2]};
  return true;
}

// One thread per face over every view of the call: world positions are read once, each view
// transforms them inline.  Triangles that need clipping or whose pixel box exceeds kInline
// pixels go to the queue as f * n_views + view.
__global__ void __launch_bounds__(128) k_raster_faces(const float* __restrict__ V, int nV,
                                                      const int32_t* __restrict__ F, int nF,
                                                      const double* __restrict__ w2c, int nv, Cam c,
                                                      unsigned* __restrict__ img,
                                                      unsigned* __restrict__ queue,
                                                      unsigned* __restrict__ q_count,
                                                      int32_t* __restrict__ status) {
  __shared__ double M[kMaxViews * 12];
  for (int k = threadIdx.x; k < nv * 12; k += blockDim.x) M[k] = w2c[k];
  __syncthreads();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nF) return;
  V3 w[3];
  if (!load_face(V, nV, F, f, w)) { *status = XRD_E_SHAPE; return; }
  const size_t plane_px = (size_t)c.H * c.W;
  for (int b = 0; b < nv; ++b) {
    const double* m = M + 12 * b;
    const V3 p0 = to_cam(m, w[0].x, w[0].y, w[0].z), p1 = to_cam(m, w[1].x, w[1].y, w[1].z),
             p2 = to_cam(m, w[2].x, w[2].y, w[2].z);
    if (p0.z < c.near && p1.z < c.near && p2.z < c.near) continue;
    if (!inside_all(c, p0) || !inside_all(c, p1) || !inside_all(c, p2)) {
      queue[atomicAdd(q_count, 1u)] = (unsigned)f * (unsigned)nv + (unsigned)b;
      continue;
    }
    Snapped s;
    if (!setup(c, p0, p1, p2, s)) continue;
    if ((s.x1 - s.x0 + 1) * (s.y1 - s.y0 + 1) > kInline) {
      queue[atomicAdd(q_count, 1u)] = (unsigned)f * (unsigned)nv + (unsigned)b;
      continue;
    }
    Plane pl;
    if (!tri_plane(c, p0, p1, p2, pl)) continue;
    unsigned* im = img + plane_px * b;
    for (int j = s.y0; j <= s.y1; ++j)
      for (int i = s.x0; i <= s.x1; ++i)
        if (covers(s, i, j)) write_depth(im, c.W, i, j, frag_depth(c, pl, i, j));
  }
}

// One warp per queued (face, view): every lane clips the triangle (the same arithmetic as the
// inline path, which the clip leaves unchanged when nothing is outside), then the lanes stride
// over each fan triangle's pixel box.
__global__ void __launch_bounds__(256) k_raster_queue(const float* __restrict__ V, int nV,
                                                      const int32_t* __restrict__ F,
                                                      const double* __restrict__ w2c, int nv, Cam c,
                                                      unsigned* __restrict__ img,
                                                      const unsigned* __restrict__ queue,
                                                      const unsigned* __restrict__ q_count) {
  const int lane = threadIdx.x & 31;
  const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned n_warps = (gridDim.x * blockDim.x) >> 5;
  const unsigned n = *q_count;
  const size_t plane_px = (size_t)c.H * c.W;
  for (unsigned e = warp; e < n; e += n_warps) {
    const unsigned ent = queue[e];
    const int f = (int)(ent / (unsigned)nv), b = (int)(ent % (unsigned)nv);
    V3 w[3];
    load_face(V, nV, F, f, w);  // indices were checked before the entry was queued
    const double* m = w2c + 12 * b;
    V3 P[kMaxPoly + 1];
#pragma unroll
    for (int k = 0; k < 3; ++k) P[k] = to_cam(m, w[k].x, w[k].y, w[k].z);
    Plane pl;
    if (!tri_plane(c, P[0], P[1], P[2], pl)) continue;
    const int np = clip_poly(c, P, 3);
    unsigned* im = img + plane_px * b;
    for (int t = 1; t + 1 < np; ++t) {
      Snapped s;
      if (!setup(c, P[0], P[t], P[t + 1], s)) continue;
      const int bw = s.x1 - s.x0 + 1;
      const int cnt = bw * (s.y1 - s.y0 + 1);
      for (int q = lane; q < cnt; q += 32) {
        const int i = s.x0 + q % bw, j = s.y0 + q / bw;
        if (covers(s, i, j)) write_depth(im, c.W, i, j, frag_depth(c, pl, i, j));
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_finish(unsigned* __restrict__ img, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = img[i];
  img[i] = k ? ~k : 0u;  // 0u is the bit pattern of 0.0f
}

// ---------------------------------------------------------------- unseen-region check ---
constexpr int kSeenViews = 32;

// check_proj in fp32 for every (point, view): cam = ((w0 x + w1 y) + w2 z) + w3 per row,
// x' = -cam_x, u' = fx x' + cx z, v' = fy y + cy z, z' = z + 1e-5, u = u' / z', v = v' / z';
// the view is seen when some point has 0 <= -z', 0 < u < W and 0 < v < H.
__global__ void __launch_bounds__(256) k_points_seen(const float* __restrict__ P, int n,
                                                     const float* __restrict__ w2c, int K,
                                                     float W, float H, float fx, float fy,
                                                     float cx, float cy,
                                                     uint8_t* __restrict__ seen) {
  __shared__ float M[kSeenViews * 12];
  const int v0 = blockIdx.y * kSeenViews;
  const int nv = min(kSeenViews, K - v0);
  for (int k = threadIdx.x; k < nv * 12; k += blockDim.x) M[k] = w2c[(size_t)v0 * 12 + k];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
  const float eps = 1e-5f;
  for (int b = 0; b < nv; ++b) {
    if (*(volatile uint8_t*)(seen + v0 + b)) continue;
    const float* m = M + 12 * b;
    const float cxp = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
    const float cyp = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], x), __fmul_rn(m[5], y)), __fmul_rn(m[6], z)), m[7]);
    const float czp = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], x), __fmul_rn(m[9], y)), __fmul_rn(m[10], z)), m[11]);
    const float xn = -cxp;
    const float zz = __fadd_rn(czp, eps);
    const float u = __fdiv_rn(__fadd_rn(__fmul_rn(fx, xn), __fmul_rn(cx, czp)), zz);
    const float v = __fdiv_rn(__fadd_rn(__fmul_rn(fy, cyp), __fmul_rn(cy, czp)), zz);
    if (0.f <= -zz && u < W && u > 0.f && v < H && v > 0.f) seen[v0 + b] = 1;
  }
}

// ---------------------------------------------------------------- per-view sums ---
constexpr int kL1Threads = 256;

// one block per view: thread t sums |gt - rec| (fp32 difference widened to f64) and the count
// over pixels t, t + 256, ... with rec > 0, then a fixed shared-memory tree
__global__ void __launch_bounds__(kL1Threads) k_depth_l1(const float* __restrict__ gt,
                                                         const float* __restrict__ rec, int n_px,
                                                         double* __restrict__ out) {
  __shared__ double sh[2][kL1Threads];
  const size_t base = (size_t)blockIdx.x * n_px;
  double s = 0.0, c = 0.0;
  for (int p = threadIdx.x; p < n_px; p += kL1Threads) {
    const float r = rec[base + p];
    if (r > 0.f) {
      s = __dadd_rn(s, (double)fabsf(__fsub_rn(gt[base + p], r)));
      c = __dadd_rn(c, 1.0);
    }
  }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = c;
  __syncthreads();
  for (int h = kL1Threads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      sh[0][threadIdx.x] = __dadd_rn(sh[0][threadIdx.x], sh[0][threadIdx.x + h]);
      sh[1][threadIdx.x] = __dadd_rn(sh[1][threadIdx.x], sh[1][threadIdx.x + h]);
    }
    __syncthreads();
  }
  if (threadIdx.x < 2) out[2 * blockIdx.x + threadIdx.x] = sh[threadIdx.x][0];
}

// ---------------------------------------------------------------- host ---
// the queue holds at most one entry per (face, view), plus its counter
struct RenderWs : Carver {
  RenderWs(void* base, int n_faces, int n_views)
      : Carver(base), count(take<unsigned>(1)),
        queue(take_last<unsigned>((size_t)n_faces * n_views)) {}
  unsigned* count;
  unsigned* queue;
};

bool camera_ok(const XrdEvalCamera& c) {
  const bool fin = std::isfinite(c.fx) && std::isfinite(c.fy) && std::isfinite(c.cx) &&
                   std::isfinite(c.cy) && std::isfinite(c.z_near) && std::isfinite(c.z_far);
  return fin && c.H >= 1 && c.W >= 1 && c.H <= XRD_EVAL_RENDER_MAX_SIDE &&
         c.W <= XRD_EVAL_RENDER_MAX_SIDE && c.fx > 0.0 && c.fy > 0.0 && c.z_near > 0.0 &&
         c.z_far > c.z_near && std::fabs(c.cx) <= 2.0 * XRD_EVAL_RENDER_MAX_SIDE &&
         std::fabs(c.cy) <= 2.0 * XRD_EVAL_RENDER_MAX_SIDE;
}

bool render_shape_ok(int n_faces, int n_views) {
  return n_faces >= 1 && n_views >= 1 && n_views <= kMaxViews &&
         (long long)n_faces * n_views <= 0x7fffffffLL;
}

}  // namespace evr
}  // namespace xrd

using namespace xrd;
using namespace xrd::evr;

extern "C" size_t xrd_eval_render_workspace_bytes(int n_faces, int n_views) {
  if (!render_shape_ok(n_faces, n_views)) return 0;
  return RenderWs(nullptr, n_faces, n_views).bytes();
}

extern "C" int xrd_eval_render_depth(const float* verts, int n_verts, const int32_t* faces,
                                     int n_faces, const double* w2c, int n_views,
                                     const XrdEvalCamera* camera, float* depth, int32_t* status,
                                     void* workspace, size_t workspace_bytes, void* stream_) {
  if (!camera) return XRD_E_NULL;
  if (n_verts < 1 || !render_shape_ok(n_faces, n_views) || !camera_ok(*camera)) return XRD_E_SHAPE;
  if (!verts || !faces || !w2c || !depth || !status || !workspace) return XRD_E_NULL;
  const RenderWs L(workspace, n_faces, n_views);
  if (int st = L.check(workspace_bytes)) return st;
  const XrdEvalCamera& k = *camera;
  const Cam c{k.H, k.W, k.fx, k.fy, k.cx, k.cy, k.z_near, k.z_far};
  cudaStream_t s = (cudaStream_t)stream_;
  const long long n_px = (long long)n_views * k.H * k.W;
  unsigned* img = reinterpret_cast<unsigned*>(depth);
  XRD_CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
  XRD_CUDA_TRY(cudaMemsetAsync(L.count, 0, sizeof(unsigned), s));
  XRD_CUDA_TRY(cudaMemsetAsync(img, 0, (size_t)n_px * sizeof(float), s));
  {
    KernelTimer timer(s);
    k_raster_faces<<<blocks(n_faces, 128), 128, 0, s>>>(verts, n_verts, faces, n_faces, w2c,
                                                         n_views, c, img, L.queue, L.count, status);
    XRD_LAUNCH_CHECK();
    k_raster_queue<<<num_sms() * 8, 256, 0, s>>>(verts, n_verts, faces, w2c, n_views, c, img,
                                                 L.queue, L.count);
    XRD_LAUNCH_CHECK();
  }
  k_finish<<<blocks(n_px), 256, 0, s>>>(img, n_px);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_debug_eval_render_queued(const void* workspace, unsigned* count, void* stream_) {
  if (!workspace || !count) return XRD_E_NULL;
  XRD_CUDA_TRY(cudaMemcpyAsync(count, workspace, sizeof(unsigned), cudaMemcpyDeviceToDevice,
                               (cudaStream_t)stream_));
  return XRD_OK;
}

extern "C" int xrd_eval_points_seen(const float* points, int n_points, const float* w2c,
                                    int n_views, const XrdEvalCamera* camera, uint8_t* seen,
                                    void* stream_) {
  if (!camera) return XRD_E_NULL;
  if (n_points < 0 || n_views < 0 || camera->H < 1 || camera->W < 1) return XRD_E_SHAPE;
  if (n_views == 0) return XRD_OK;
  if (!w2c || !seen || (n_points > 0 && !points)) return XRD_E_NULL;
  cudaStream_t s = (cudaStream_t)stream_;
  XRD_CUDA_TRY(cudaMemsetAsync(seen, 0, (size_t)n_views, s));
  if (n_points == 0) return XRD_OK;
  const XrdEvalCamera& k = *camera;
  const dim3 grid(blocks(n_points), (unsigned)((n_views + kSeenViews - 1) / kSeenViews));
  k_points_seen<<<grid, 256, 0, s>>>(points, n_points, w2c, n_views, (float)k.W, (float)k.H,
                                     (float)k.fx, (float)k.fy, (float)k.cx, (float)k.cy, seen);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_eval_depth_l1(const float* gt, const float* rec, int n_views, int n_pixels,
                                 double* out, void* stream_) {
  if (n_views < 0 || n_pixels < 0) return XRD_E_SHAPE;
  if (n_views == 0) return XRD_OK;
  if (!gt || !rec || !out) return XRD_E_NULL;
  k_depth_l1<<<n_views, kL1Threads, 0, (cudaStream_t)stream_>>>(gt, rec, n_pixels, out);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
