// ds-eval reconstruction metrics on the device (sm_90a): area-weighted surface sampling, an exact
// nearest-neighbour index with unbounded and radius-bounded queries, deterministic float64
// reductions and the float64 rigid transform.
//
// Replaces (reference @ f0366f20):
//   scripts/utils/eval_recon.py:29-47    completion_ratio / accuracy / completion (cKDTree)
//   scripts/utils/eval_recon.py:93-136   calc_3d_metric: trimesh.sample.sample_surface, ICP
//   third_party/evaluate_3d_reconstruction_lib/.../evaluate_3d_reconstruction.py:50-276
//                                        run_evaluation: sample_points_uniformly, ICP,
//                                        compute_point_cloud_distance
// Semantics (fixed here, documented in include/xrdslam_b200.h under xrd_eval_* / xrd_nn_*):
// every fp32 / fp64 operation is rounded to nearest in the order written (explicit intrinsics, no
// contraction); a query's result is the minimum of (d^2, id) over the candidates, so it does not
// depend on traversal order or launch split; reductions use fixed chunks and a fixed final order.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <cmath>

#include "common.cuh"

namespace xrd {
namespace eval {

thread_local unsigned long long* g_nn_counters = nullptr;

constexpr int kChunk = XRD_EVAL_AREA_CHUNK;    // faces per sequential prefix-sum chunk
constexpr int kRedChunk = XRD_EVAL_RED_CHUNK;  // elements per reduction partial
constexpr int kRedThreads = 256;

unsigned blocks(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

// ---------------------------------------------------------------- surface sampling ---
__device__ __forceinline__ double face_area(const float* __restrict__ V, int a, int b, int c) {
  const double ax = V[3 * a], ay = V[3 * a + 1], az = V[3 * a + 2];
  const double e1x = __dsub_rn(V[3 * b], ax), e1y = __dsub_rn(V[3 * b + 1], ay),
               e1z = __dsub_rn(V[3 * b + 2], az);
  const double e2x = __dsub_rn(V[3 * c], ax), e2y = __dsub_rn(V[3 * c + 1], ay),
               e2z = __dsub_rn(V[3 * c + 2], az);
  const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz));
  return __dmul_rn(0.5, __dsqrt_rn(n2));
}

__global__ void __launch_bounds__(256) k_check_verts(const float* __restrict__ V, int n,
                                                     int32_t* status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 3LL * n && !isfinite(V[i])) *status = XRD_E_SHAPE;
}

// one thread per chunk: sequential area prefix inside the chunk, chunk total to tot[c]
__global__ void __launch_bounds__(128) k_area_chunks(const float* __restrict__ V, int nV,
                                                     const int32_t* __restrict__ F, int nF,
                                                     double* __restrict__ cum,
                                                     double* __restrict__ tot, int32_t* status) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = c * kChunk;
  if (b >= nF) return;
  const int e = min(nF, b + kChunk);
  double s = 0.0;
  bool bad = false;
  for (int f = b; f < e; ++f) {
    const int i0 = F[3 * f], i1 = F[3 * f + 1], i2 = F[3 * f + 2];
    if (i0 < 0 || i0 >= nV || i1 < 0 || i1 >= nV || i2 < 0 || i2 >= nV) {
      bad = true;
    } else {
      s = __dadd_rn(s, face_area(V, i0, i1, i2));
    }
    cum[f] = s;
  }
  tot[c] = s;
  if (bad) *status = XRD_E_SHAPE;
}

// single thread: exclusive sequential sum of the chunk totals; total area must be finite and > 0
__global__ void k_area_offsets(double* tot, int n_chunks, double* total, int32_t* status) {
  if (threadIdx.x || blockIdx.x) return;
  double s = 0.0;
  for (int c = 0; c < n_chunks; ++c) {
    const double t = tot[c];
    tot[c] = s;
    s = __dadd_rn(s, t);
  }
  *total = s;
  if (!(s > 0.0) || !isfinite(s)) *status = XRD_E_SHAPE;
}

__global__ void __launch_bounds__(256) k_area_add(double* __restrict__ cum, int nF,
                                                  const double* __restrict__ off) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nF) cum[f] = __dadd_rn(off[f / kChunk], cum[f]);
}

// first index i with cum[i] >= x (numpy.searchsorted side='left'), clamped to n - 1
__device__ __forceinline__ int search_left(const double* __restrict__ cum, int n, double x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (cum[m] < x) lo = m + 1; else hi = m;
  }
  return min(lo, n - 1);
}

__device__ __forceinline__ void uniforms(const float* __restrict__ U, int per, uint64_t seed,
                                         int i, float u[4]) {
  if (U) {
    for (int j = 0; j < per; ++j) u[j] = U[(size_t)i * per + j];
  } else {
    philox4(seed, (uint64_t)i, u);
  }
}

// mode 0 (trimesh sample_surface): face = searchsorted(cum, u0 * total); (u1, u2) folded when
// u1 + u2 > 1; p = v0 + (u1 * (v1 - v0) + u2 * (v2 - v0)).
// mode 1 (open3d sample_points_uniformly): face t owns [round(cum[t-1] / total * n),
// round(cum[t] / total * n)); a = 1 - sqrt(r1), b = sqrt(r1) (1 - r2), c = sqrt(r1) r2;
// p = (a v0 + b v1) + c v2.
__global__ void __launch_bounds__(256) k_sample(const float* __restrict__ V,
                                                const int32_t* __restrict__ F, int nF,
                                                const double* __restrict__ cum,
                                                const double* __restrict__ total, int mode, int n,
                                                const float* __restrict__ U, uint64_t seed,
                                                const int32_t* __restrict__ status,
                                                float* __restrict__ out,
                                                int32_t* __restrict__ face_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || *status != XRD_OK) return;
  const double S = *total;
  float u[4];
  uniforms(U, mode == 0 ? 3 : 2, seed, i, u);
  int f;
  float w0, w1, w2;
  if (mode == 0) {
    f = search_left(cum, nF, __dmul_rn((double)u[0], S));
    float a = u[1], b = u[2];
    if (__fadd_rn(a, b) > 1.f) { a = fabsf(__fsub_rn(a, 1.f)); b = fabsf(__fsub_rn(b, 1.f)); }
    w1 = a; w2 = b; w0 = 0.f;
  } else {
    // first t with round(cum[t] / S * n) > i
    int lo = 0, hi = nF;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (round(__dmul_rn(__ddiv_rn(cum[m], S), (double)n)) > (double)i) hi = m; else lo = m + 1;
    }
    f = min(lo, nF - 1);
    const float sr = __fsqrt_rn(u[0]);
    w0 = __fsub_rn(1.f, sr);
    w1 = __fmul_rn(sr, __fsub_rn(1.f, u[1]));
    w2 = __fmul_rn(sr, u[1]);
  }
  const int i0 = F[3 * f], i1 = F[3 * f + 1], i2 = F[3 * f + 2];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float p0 = V[3 * i0 + d], p1 = V[3 * i1 + d], p2 = V[3 * i2 + d];
    float p;
    if (mode == 0) {
      p = __fadd_rn(p0, __fadd_rn(__fmul_rn(w1, __fsub_rn(p1, p0)),
                                  __fmul_rn(w2, __fsub_rn(p2, p0))));
    } else {
      p = __fadd_rn(__fadd_rn(__fmul_rn(w0, p0), __fmul_rn(w1, p1)), __fmul_rn(w2, p2));
    }
    out[(size_t)3 * i + d] = p;
  }
  if (face_out) face_out[i] = f;
}

// ---------------------------------------------------------------- nearest neighbour ---
__device__ __forceinline__ int clampi(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

__device__ __forceinline__ int cell_of(const XrdNnIndex& I, float x, float y, float z) {
  const int cx = clampi((int)floorf(__fmul_rn(__fsub_rn(x, I.origin[0]), I.inv_h)), I.dims[0] - 1);
  const int cy = clampi((int)floorf(__fmul_rn(__fsub_rn(y, I.origin[1]), I.inv_h)), I.dims[1] - 1);
  const int cz = clampi((int)floorf(__fmul_rn(__fsub_rn(z, I.origin[2]), I.inv_h)), I.dims[2] - 1);
  return (cz * I.dims[1] + cy) * I.dims[0] + cx;
}

__global__ void __launch_bounds__(256) k_nn_keys(const float* __restrict__ P, int n, XrdNnIndex I,
                                                 int* __restrict__ keys, int* __restrict__ ids,
                                                 int* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = cell_of(I, P[3 * i], P[3 * i + 1], P[3 * i + 2]);
  keys[i] = c;
  ids[i] = i;
  atomicAdd(counts + c, 1);
}

__global__ void __launch_bounds__(256) k_nn_gather(const float* __restrict__ P, int n,
                                                   const int* __restrict__ ids,
                                                   float4* __restrict__ sorted) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = ids[i];
  sorted[i] = make_float4(P[3 * j], P[3 * j + 1], P[3 * j + 2], __int_as_float(j));
}

// level dims: ceil(dims / 2^l)
__device__ __forceinline__ int ldim(int d, int l) { return ((d - 1) >> l) + 1; }

__global__ void __launch_bounds__(256) k_nn_occupancy(XrdNnIndex I, const int* __restrict__ counts,
                                                      uint8_t* __restrict__ occ) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= I.n_cells || counts[c] == 0) return;
  const int x = c % I.dims[0], y = (c / I.dims[0]) % I.dims[1], z = c / (I.dims[0] * I.dims[1]);
  for (int l = 1; l <= I.n_levels; ++l) {
    const int nx = ldim(I.dims[0], l), ny = ldim(I.dims[1], l);
    occ[I.level_off[l] + ((z >> l) * ny + (y >> l)) * nx + (x >> l)] = 1;
  }
}

// exact nearest target of one query: depth-first over the implicit octree of the grid, children
// in the order (c ^ octant of q), a 4-bit next-child counter per level packed in one word;
// a node is pruned when its padded box's lower bound exceeds the best d^2 with a margin that
// rounding cannot cross, so every candidate with d^2 <= best is scanned.
__global__ void __launch_bounds__(256) k_nn_query(XrdNnIndex I, const float* __restrict__ Q, int nq,
                                                  float r2, float* __restrict__ dist,
                                                  int32_t* __restrict__ ids,
                                                  unsigned long long* counters) {
  const int qi = blockIdx.x * blockDim.x + threadIdx.x;
  if (qi >= nq) return;
  const float qx = Q[3 * qi], qy = Q[3 * qi + 1], qz = Q[3 * qi + 2];
  const float4* __restrict__ S = reinterpret_cast<const float4*>(I.sorted);
  float best = r2;
  int bid = 0x7fffffff;
  unsigned nodes = 0, pts = 0;
  int l = I.n_levels, cx = 0, cy = 0, cz = 0;
  unsigned long long ctr = 0;
  const float margin = 0.99998f;  // 1 - 2^-15.6: far above the relative rounding of d^2 and lb
  while (true) {
    if (l == 0) {
      const int c = (cz * I.dims[1] + cy) * I.dims[0] + cx;
      const int e = I.cell_ptr[c + 1];
      for (int k = I.cell_ptr[c]; k < e; ++k) {
        const float4 p = __ldg(S + k);
        const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)),
                                   __fmul_rn(dz, dz));
        const int id = __float_as_int(p.w);
        if (d2 < best || (d2 == best && id < bid)) { best = d2; bid = id; }
      }
      pts += (unsigned)(e - I.cell_ptr[c]);
      if (I.n_levels == 0) break;
      l = 1; cx >>= 1; cy >>= 1; cz >>= 1;
    }
    const int sh = 4 * (l - 1);
    const int c = (int)((ctr >> sh) & 15);
    if (c == 8) {
      if (l == I.n_levels) break;
      ctr &= ~(15ull << sh);
      ++l; cx >>= 1; cy >>= 1; cz >>= 1;
      continue;
    }
    ctr += 1ull << sh;
    // node centre decides the near-first order of its children
    const float half = __fmul_rn(I.h, (float)(1 << (l - 1)));
    const int oct = (qx >= __fadd_rn(I.origin[0], __fmul_rn(half, (float)(2 * cx + 1))) ? 1 : 0) |
                    (qy >= __fadd_rn(I.origin[1], __fmul_rn(half, (float)(2 * cy + 1))) ? 2 : 0) |
                    (qz >= __fadd_rn(I.origin[2], __fmul_rn(half, (float)(2 * cz + 1))) ? 4 : 0);
    const int o = c ^ oct;
    const int nx = 2 * cx + (o & 1), ny = 2 * cy + ((o >> 1) & 1), nz = 2 * cz + (o >> 2);
    const int lc = l - 1;
    const int dx_ = ldim(I.dims[0], lc), dy_ = ldim(I.dims[1], lc), dz_ = ldim(I.dims[2], lc);
    if (nx >= dx_ || ny >= dy_ || nz >= dz_) continue;
    const int lin = (nz * dy_ + ny) * dx_ + nx;
    if (lc == 0 ? I.cell_ptr[lin + 1] == I.cell_ptr[lin] : !I.occ[I.level_off[lc] + lin]) continue;
    // lower bound of d^2 over the child's padded box
    float lb = 0.f;
    {
      const float w = __fmul_rn(I.h, (float)(1 << lc));
      const float lo0 = __fsub_rn(__fadd_rn(I.origin[0], __fmul_rn(w, (float)nx)), I.pad);
      const float lo1 = __fsub_rn(__fadd_rn(I.origin[1], __fmul_rn(w, (float)ny)), I.pad);
      const float lo2 = __fsub_rn(__fadd_rn(I.origin[2], __fmul_rn(w, (float)nz)), I.pad);
      const float g0 = fmaxf(fmaxf(__fsub_rn(lo0, qx), __fsub_rn(qx, __fadd_rn(__fadd_rn(lo0, w), __fmul_rn(2.f, I.pad)))), 0.f);
      const float g1 = fmaxf(fmaxf(__fsub_rn(lo1, qy), __fsub_rn(qy, __fadd_rn(__fadd_rn(lo1, w), __fmul_rn(2.f, I.pad)))), 0.f);
      const float g2 = fmaxf(fmaxf(__fsub_rn(lo2, qz), __fsub_rn(qz, __fadd_rn(__fadd_rn(lo2, w), __fmul_rn(2.f, I.pad)))), 0.f);
      lb = __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(g0, g0), __fmul_rn(g1, g1)), __fmul_rn(g2, g2)),
                     margin);
    }
    if (lb > best) continue;
    ++nodes;
    l = lc; cx = nx; cy = ny; cz = nz;
  }
  const bool found = bid != 0x7fffffff;
  dist[qi] = found ? __fsqrt_rn(best) : INFINITY;
  ids[qi] = found ? bid : -1;
  if (counters) {
    atomicAdd(counters, (unsigned long long)nodes);
    atomicAdd(counters + 1, (unsigned long long)pts);
  }
}

// ---------------------------------------------------------------- reductions ---
// Per partial p: elements [p * kRedChunk, (p + 1) * kRedChunk) in thread-strided order, then a
// fixed shared-memory tree; the final kernel sums the partials in index order.
template <int K, class Fn>
__device__ __forceinline__ void reduce_block(int n, Fn fn, double* __restrict__ part) {
  __shared__ double sh[K][kRedThreads];
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  const int b = blockIdx.x * kRedChunk;
  const int e = min(n, b + kRedChunk);
  for (int i = b + threadIdx.x; i < e; i += kRedThreads) fn(i, acc);
#pragma unroll
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int s = kRedThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k)
        sh[k][threadIdx.x] = __dadd_rn(sh[k][threadIdx.x], sh[k][threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x < K) part[(size_t)blockIdx.x * K + threadIdx.x] = sh[threadIdx.x][0];
}

__global__ void __launch_bounds__(kRedThreads) k_dist_partials(const float* __restrict__ d, int n,
                                                              float tau, double* part) {
  reduce_block<3>(n, [&](int i, double* acc) {
    const double x = d[i];
    acc[0] = __dadd_rn(acc[0], x);
    acc[1] = __dadd_rn(acc[1], __dmul_rn(x, x));
    acc[2] = __dadd_rn(acc[2], d[i] < tau ? 1.0 : 0.0);
  }, part);
}

// fields: count, sum s (3), sum t (3), sum s t^T (9, row-major [s][t]), sum d^2
__global__ void __launch_bounds__(kRedThreads) k_icp_partials(const float* __restrict__ src,
                                                             const float* __restrict__ tgt,
                                                             const int32_t* __restrict__ ids,
                                                             const float* __restrict__ d, int n,
                                                             double* part) {
  reduce_block<17>(n, [&](int i, double* acc) {
    const int j = ids[i];
    if (j < 0) return;
    const double s[3] = {src[3 * i], src[3 * i + 1], src[3 * i + 2]};
    const double t[3] = {tgt[3 * j], tgt[3 * j + 1], tgt[3 * j + 2]};
    acc[0] = __dadd_rn(acc[0], 1.0);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      acc[1 + a] = __dadd_rn(acc[1 + a], s[a]);
      acc[4 + a] = __dadd_rn(acc[4 + a], t[a]);
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[7 + 3 * a + b] = __dadd_rn(acc[7 + 3 * a + b], __dmul_rn(s[a], t[b]));
    }
    const double x = d[i];
    acc[16] = __dadd_rn(acc[16], __dmul_rn(x, x));
  }, part);
}

__global__ void k_final(const double* __restrict__ part, int n_part, int K, double* out) {
  const int k = threadIdx.x;
  if (k >= K) return;
  double s = 0.0;
  for (int p = 0; p < n_part; ++p) s = __dadd_rn(s, part[(size_t)p * K + k]);
  out[k] = s;
}

// ---------------------------------------------------------------- transform ---
struct Rigid { double m[12]; };

__global__ void __launch_bounds__(256) k_transform(const float* __restrict__ in, int n, Rigid T,
                                                   float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = in[3 * i], y = in[3 * i + 1], z = in[3 * i + 2];
  float r[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* R = T.m + 4 * a;
    r[a] = __double2float_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[0], x), __dmul_rn(R[1], y)),
                                                 __dmul_rn(R[2], z)),
                                       R[3]));
  }
  out[3 * i] = r[0]; out[3 * i + 1] = r[1]; out[3 * i + 2] = r[2];
}

// ---------------------------------------------------------------- host helpers ---
int n_chunks(int nF) { return (nF + kChunk - 1) / kChunk; }
int n_partials(int n) { return n <= 0 ? 1 : (n + kRedChunk - 1) / kRedChunk; }

struct NnWs {
  size_t keys, keys2, ids, ids2, counts, sort, sort_bytes, scan, scan_bytes, total;
};

NnWs nn_ws(int n, int n_cells) {
  NnWs L;
  size_t q = 0;
  auto take = [&](size_t b) { size_t o = q; q += align_up(b, 256); return o; };
  L.keys = take((size_t)n * 4);
  L.keys2 = take((size_t)n * 4);
  L.ids = take((size_t)n * 4);
  L.ids2 = take((size_t)n * 4);
  L.counts = take((size_t)(n_cells + 1) * 4);
  L.sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, L.sort_bytes, (const int*)nullptr, (int*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n);
  L.sort = take(L.sort_bytes);
  L.scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, L.scan_bytes, (const int*)nullptr, (int*)nullptr,
                                n_cells + 1);
  L.scan = take(L.scan_bytes);
  L.total = q;
  return L;
}

long long cells_for(const double ext[3], double h, int dims[3]) {
  long long c = 1;
  for (int a = 0; a < 3; ++a) {
    const double d = floor(ext[a] / h) + 1.0;
    if (d > (double)XRD_NN_MAX_DIM) return -1;
    dims[a] = (int)d;
    c *= dims[a];
  }
  return c;
}

bool index_ok(const XrdNnIndex& I) {
  return I.n_points >= 1 && I.n_cells >= 1 && I.n_levels >= 0 && I.n_levels < XRD_NN_MAX_LEVELS &&
         I.h > 0.f && I.cell_ptr && I.sorted && (I.n_levels == 0 || I.occ);
}

}  // namespace eval
}  // namespace xrd

using namespace xrd;
using namespace xrd::eval;

extern "C" size_t xrd_eval_surface_workspace_bytes(int n_faces) {
  if (n_faces < 1) return 0;
  return align_up((size_t)n_chunks(n_faces) * sizeof(double), 256) + 256;
}

extern "C" int xrd_eval_surface_prepare(const float* verts, int n_verts, const int32_t* faces,
                                        int n_faces, double* cum, double* total, int32_t* status,
                                        void* workspace, size_t workspace_bytes, void* stream_) {
  if (n_faces < 1 || n_verts < 1) return XRD_E_SHAPE;
  if (!verts || !faces || !cum || !total || !status || !workspace) return XRD_E_NULL;
  if (workspace_bytes < xrd_eval_surface_workspace_bytes(n_faces)) return XRD_E_WORKSPACE;
  cudaStream_t s = (cudaStream_t)stream_;
  double* tot = reinterpret_cast<double*>(workspace);
  const int nc = n_chunks(n_faces);
  XRD_CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
  k_check_verts<<<blocks(3LL * n_verts), 256, 0, s>>>(verts, n_verts, status);
  XRD_LAUNCH_CHECK();
  k_area_chunks<<<blocks(nc, 128), 128, 0, s>>>(verts, n_verts, faces, n_faces, cum, tot, status);
  XRD_LAUNCH_CHECK();
  k_area_offsets<<<1, 32, 0, s>>>(tot, nc, total, status);
  XRD_LAUNCH_CHECK();
  k_area_add<<<blocks(n_faces), 256, 0, s>>>(cum, n_faces, tot);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_eval_sample_surface(const float* verts, const int32_t* faces, int n_faces,
                                       const double* cum, const double* total,
                                       const int32_t* status, int mode, int n_samples,
                                       const float* uniforms, uint64_t seed, float* out,
                                       int32_t* face_ids, void* stream_) {
  if (n_faces < 1 || n_samples < 0 || (mode != XRD_EVAL_TRIMESH && mode != XRD_EVAL_OPEN3D))
    return XRD_E_SHAPE;
  if (!verts || !faces || !cum || !total || !status || (n_samples > 0 && !out)) return XRD_E_NULL;
  if (n_samples == 0) return XRD_OK;
  cudaStream_t s = (cudaStream_t)stream_;
  k_sample<<<blocks(n_samples), 256, 0, s>>>(verts, faces, n_faces, cum, total, mode, n_samples,
                                              uniforms, seed, status, out, face_ids);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_nn_layout(int n_points, const double* bbox_min, const double* bbox_max,
                             XrdNnIndex* index) {
  if (!bbox_min || !bbox_max || !index) return XRD_E_NULL;
  if (n_points < 1 || n_points > (1 << 30)) return XRD_E_SHAPE;
  double ext[3], emax = 0.0, mabs = 0.0;
  for (int a = 0; a < 3; ++a) {
    if (!std::isfinite(bbox_min[a]) || !std::isfinite(bbox_max[a]) || bbox_max[a] < bbox_min[a])
      return XRD_E_SHAPE;
    ext[a] = bbox_max[a] - bbox_min[a];
    emax = fmax(emax, ext[a]);
    mabs = fmax(mabs, fmax(fabs(bbox_min[a]), fabs(bbox_max[a])));
  }
  const long long target = 2LL * n_points;
  int dims[3] = {1, 1, 1};
  double h = 1.0;
  if (emax > 0.0) {
    // smallest h (bisection, 64 steps) with at most 2 N cells and XRD_NN_MAX_DIM per axis
    double lo = emax / (double)(XRD_NN_MAX_DIM - 1), hi = emax * 1.000001;
    for (int it = 0; it < 64; ++it) {
      const double m = 0.5 * (lo + hi);
      int d[3];
      const long long c = cells_for(ext, m, d);
      if (c >= 1 && c <= target) hi = m; else lo = m;
    }
    h = hi;
    cells_for(ext, h, dims);
  }
  XrdNnIndex& I = *index;
  I.n_points = n_points;
  for (int a = 0; a < 3; ++a) {
    I.origin[a] = (float)bbox_min[a];
    I.dims[a] = dims[a];
  }
  I.h = (float)h;
  I.inv_h = (float)(1.0 / (double)I.h);
  // binning and box corners are fp32 around |x| <= mabs + emax: pad far beyond their rounding
  I.pad = (float)(1e-4 * h + 64.0 * (mabs + emax) * 1.1920928955078125e-07);
  I.n_cells = dims[0] * dims[1] * dims[2];
  int L = 0;
  while (((dims[0] - 1) >> L) || ((dims[1] - 1) >> L) || ((dims[2] - 1) >> L)) ++L;
  I.n_levels = L;
  long long off = 0;
  for (int l = 0; l < XRD_NN_MAX_LEVELS; ++l) I.level_off[l] = 0;
  for (int l = 1; l <= L; ++l) {
    I.level_off[l] = (int)off;
    off += (long long)(((dims[0] - 1) >> l) + 1) * (((dims[1] - 1) >> l) + 1) *
           (((dims[2] - 1) >> l) + 1);
  }
  I.occ_bytes = (int)off;
  return XRD_OK;
}

extern "C" size_t xrd_nn_build_workspace_bytes(const XrdNnIndex* index) {
  if (!index || index->n_points < 1 || index->n_cells < 1) return 0;
  return nn_ws(index->n_points, index->n_cells).total;
}

extern "C" int xrd_nn_build(const float* points, const XrdNnIndex* index, void* workspace,
                            size_t workspace_bytes, void* stream_) {
  if (!points || !index || !workspace) return XRD_E_NULL;
  const XrdNnIndex I = *index;
  if (!index_ok(I)) return I.cell_ptr && I.sorted ? XRD_E_SHAPE : XRD_E_NULL;
  const NnWs L = nn_ws(I.n_points, I.n_cells);
  if (workspace_bytes < L.total) return XRD_E_WORKSPACE;
  cudaStream_t s = (cudaStream_t)stream_;
  char* ws = reinterpret_cast<char*>(workspace);
  int* keys = reinterpret_cast<int*>(ws + L.keys);
  int* keys2 = reinterpret_cast<int*>(ws + L.keys2);
  int* ids = reinterpret_cast<int*>(ws + L.ids);
  int* ids2 = reinterpret_cast<int*>(ws + L.ids2);
  int* counts = reinterpret_cast<int*>(ws + L.counts);
  const int n = I.n_points;
  XRD_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)(I.n_cells + 1) * 4, s));
  k_nn_keys<<<blocks(n), 256, 0, s>>>(points, n, I, keys, ids, counts);
  XRD_LAUNCH_CHECK();
  int end_bit = 1;
  while (end_bit < 31 && (I.n_cells - 1) >> end_bit) ++end_bit;
  size_t sb = L.sort_bytes;
  XRD_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.sort, sb, keys, keys2, ids, ids2, n, 0,
                                               end_bit, s));
  sb = L.scan_bytes;
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + L.scan, sb, counts,
                                             const_cast<int32_t*>(I.cell_ptr), I.n_cells + 1, s));
  k_nn_gather<<<blocks(n), 256, 0, s>>>(points, n, ids2, reinterpret_cast<float4*>(
                                                              const_cast<float*>(I.sorted)));
  XRD_LAUNCH_CHECK();
  if (I.n_levels > 0) {
    uint8_t* occ = const_cast<uint8_t*>(I.occ);
    XRD_CUDA_TRY(cudaMemsetAsync(occ, 0, (size_t)I.occ_bytes, s));
    k_nn_occupancy<<<blocks(I.n_cells), 256, 0, s>>>(I, counts, occ);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}

extern "C" int xrd_nn_query(const XrdNnIndex* index, const float* queries, int n_queries,
                            float radius, float* dist, int32_t* ids, void* stream_) {
  if (!index) return XRD_E_NULL;
  if (n_queries < 0 || !index_ok(*index) || radius != radius) return XRD_E_SHAPE;
  if (n_queries == 0) return XRD_OK;
  if (!queries || !dist || !ids) return XRD_E_NULL;
  const float r2 = radius > 0.f && isfinite(radius) ? radius * radius : INFINITY;
  cudaStream_t s = (cudaStream_t)stream_;
  k_nn_query<<<blocks(n_queries), 256, 0, s>>>(*index, queries, n_queries, r2, dist, ids,
                                                g_nn_counters);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_debug_nn_counters(unsigned long long* counters) {
  g_nn_counters = counters;
  return XRD_OK;
}

extern "C" size_t xrd_eval_reduce_workspace_bytes(int n) {
  if (n < 0) return 0;
  return (size_t)n_partials(n) * 17 * sizeof(double);
}

extern "C" int xrd_eval_dist_stats(const float* dist, int n, float tau, double* out,
                                   void* workspace, size_t workspace_bytes, void* stream_) {
  if (!out || !workspace || (n > 0 && !dist)) return XRD_E_NULL;
  if (n < 0) return XRD_E_SHAPE;
  if (workspace_bytes < xrd_eval_reduce_workspace_bytes(n)) return XRD_E_WORKSPACE;
  cudaStream_t s = (cudaStream_t)stream_;
  double* part = reinterpret_cast<double*>(workspace);
  const int np = n_partials(n);
  k_dist_partials<<<np, kRedThreads, 0, s>>>(dist, n, tau, part);
  XRD_LAUNCH_CHECK();
  k_final<<<1, 32, 0, s>>>(part, np, 3, out);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_eval_icp_stats(const float* src, const float* tgt, const int32_t* ids,
                                  const float* dist, int n, double* out, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  if (!out || !workspace || (n > 0 && (!src || !tgt || !ids || !dist))) return XRD_E_NULL;
  if (n < 0) return XRD_E_SHAPE;
  if (workspace_bytes < xrd_eval_reduce_workspace_bytes(n)) return XRD_E_WORKSPACE;
  cudaStream_t s = (cudaStream_t)stream_;
  double* part = reinterpret_cast<double*>(workspace);
  const int np = n_partials(n);
  k_icp_partials<<<np, kRedThreads, 0, s>>>(src, tgt, ids, dist, n, part);
  XRD_LAUNCH_CHECK();
  k_final<<<1, 32, 0, s>>>(part, np, 17, out);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_eval_transform(const float* points, int n, const double* T, float* out,
                                  void* stream_) {
  if (!T) return XRD_E_NULL;
  if (n < 0) return XRD_E_SHAPE;
  if (n == 0) return XRD_OK;
  if (!points || !out) return XRD_E_NULL;
  Rigid R;
  for (int k = 0; k < 12; ++k) R.m[k] = T[k];
  cudaStream_t s = (cudaStream_t)stream_;
  k_transform<<<blocks(n), 256, 0, s>>>(points, n, R, out);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
