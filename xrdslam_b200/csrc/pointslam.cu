// Point-SLAM render-and-optimise step, stages 'geometry' and 'color' (sm_90a): exact hash-grid kNN, inverse-
// distance feature interpolation over the neural point cloud, Fourier MLP, normalised occupancy
// compositing, losses and backward.
//
// Replaces (reference @ f0366f20):
//   slam/model_components/neural_point_cloud.py:223-282 find_neighbors_faiss (faiss-gpu IVFFlat
//       through host numpy round trips -> exact in-kernel radius kNN, SURVEY A.4)
//   slam/model_components/decoder_pointslam.py:162-273 MLP_geometry.get_feature_at_pos / forward
//   slam/models/conv_onet_pointslam.py:311-461 render_batch_ray, :144-195 get_loss_dict
//   slam/model_components/utils.py:247-295 raw2outputs_nerf_color2
// The 5x32 Fourier MLP is the NICE decoder with sin(2 pi p B) and an externally supplied
// feature (nice::launch_decoder).
#include <float.h>
#include <math.h>

#include "mlp.cuh"
#include "nice.cuh"

namespace xrd {
namespace point {

constexpr int KNN = 8;
constexpr int CD = 32;

__device__ __forceinline__ uint32_t bucket_of(int ix, int iy, int iz, int table) {
  return ((uint32_t)ix * 73856093u ^ (uint32_t)iy * 19349663u ^ (uint32_t)iz * 83492791u) &
         (uint32_t)(table - 1);
}
__device__ __forceinline__ float sqdist(const float a[3], const float* b) {
  const float dx = __fsub_rn(b[0], a[0]), dy = __fsub_rn(b[1], a[1]), dz = __fsub_rn(b[2], a[2]);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

struct KnnParams {
  XrdPointIndex ix;
  const float* q;       // [P][3]  or NULL: derive from rays / z
  const float *rays_o, *rays_d, *z;
  int S;
  const float* radius;  // per query (stride 1) or per ray (stride S via division)
  int radius_div;       // query index / radius_div selects the radius
  int P;
  float* D; int* I; int* nn;
};

__device__ __forceinline__ void query_point(const KnnParams& K, int p, float out[3]) {
  if (K.q) { out[0] = K.q[p * 3]; out[1] = K.q[p * 3 + 1]; out[2] = K.q[p * 3 + 2]; return; }
  const int r = p / K.S;
  const float z = K.z[p];
#pragma unroll
  for (int d = 0; d < 3; ++d)
    out[d] = __fadd_rn(K.rays_o[r * 3 + d], __fmul_rn(K.rays_d[r * 3 + d], z));
}

// exact radius-limited 8-NN, ascending (D, id); missing entries: id -1, D = FLT_MAX (faiss).
// KG = 8 lanes cooperate on a query: lane `sub` scans cells sub, sub + 8, .. of the (<= 27-cell)
// neighbourhood -- the scan is a chain of dependent loads (cell range -> id -> position), so the
// memory-level parallelism has to come from threads, and one thread per query leaves the
// machine at 8 % occupancy for a 25 000-query batch -- then the 8 sorted lists are merged by
// three butterfly rounds of shuffles.  (D, id) is a strict total order, so the result does not
// depend on the scan order: bit-identical to the one-thread-per-query version.
constexpr int KG = 8;

__device__ __forceinline__ void knn_insert(float (&bd)[KNN], int (&bi)[KNN], float cd, int ci) {
  if (!(cd < bd[KNN - 1] || (cd == bd[KNN - 1] && (ci < bi[KNN - 1] || bi[KNN - 1] < 0)))) return;
#pragma unroll
  for (int t = 0; t < KNN; ++t) {
    const bool before = cd < bd[t] || (cd == bd[t] && (ci < bi[t] || bi[t] < 0));
    if (before) { const float td = bd[t]; const int ti = bi[t]; bd[t] = cd; bi[t] = ci; cd = td; ci = ti; }
  }
}

// The hash-grid cell walk: visit(id, x) for every cloud point in the cells c0, c0 + cstep, ..
// of the box [q - r, q + r]; a visit returning true ends the walk.
template <class Visit>
__device__ __forceinline__ void walk_cells(const XrdPointIndex& ix, const float q[3], float r,
                                           int c0, int cstep, Visit&& visit) {
  const float inv = 1.0f / ix.cell;
  int lo[3], n[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    lo[d] = (int)floorf((q[d] - r) * inv);
    n[d] = (int)floorf((q[d] + r) * inv) - lo[d] + 1;
  }
  const int ncell = n[0] * n[1] * n[2];
  for (int c = c0; c < ncell; c += cstep) {
    const int ixx = lo[0] + c % n[0], iy = lo[1] + (c / n[0]) % n[1], iz = lo[2] + c / (n[0] * n[1]);
    const uint32_t b = bucket_of(ixx, iy, iz, ix.table_size);
    const int s = ix.cell_start[b], e = ix.cell_end[b];
    for (int j = s; j < e; ++j) {
      const int id = ix.sorted_ids[j];
      const float* x = ix.pos + (size_t)id * 3;
      // a bucket can hold several cells: accept the point only in its own cell's turn
      if ((int)floorf(x[0] * inv) != ixx || (int)floorf(x[1] * inv) != iy ||
          (int)floorf(x[2] * inv) != iz)
        continue;
      if (visit(id, x)) return;
    }
  }
}

__global__ void __launch_bounds__(128) k_knn(const KnnParams K) {
  const int gt = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = gt / KG, sub = gt % KG;
  const bool valid = p < K.P;
  float bd[KNN]; int bi[KNN];
#pragma unroll
  for (int j = 0; j < KNN; ++j) { bd[j] = FLT_MAX; bi[j] = -1; }
  float r2 = 0.f;
  if (valid) {
    float q[3];
    query_point(K, p, q);
    const float r = K.radius[p / K.radius_div];
    r2 = r * r;
    walk_cells(K.ix, q, r, sub, KG, [&](int id, const float* x) {
      const float d2 = sqdist(q, x);
      if (!(d2 > r2)) knn_insert(bd, bi, d2, id);
      return false;
    });
  }
  // butterfly merge inside the group of KG lanes (all 32 lanes take part in the shuffles)
#pragma unroll
  for (int m = 1; m < KG; m <<= 1) {
    float od[KNN]; int oi[KNN];
#pragma unroll
    for (int j = 0; j < KNN; ++j) {
      od[j] = __shfl_xor_sync(0xffffffffu, bd[j], m);
      oi[j] = __shfl_xor_sync(0xffffffffu, bi[j], m);
    }
#pragma unroll
    for (int j = 0; j < KNN; ++j)
      if (oi[j] >= 0) knn_insert(bd, bi, od[j], oi[j]);
  }
  if (!valid) return;
  // every lane of the group now holds the full list: lane `sub` writes entry `sub`
  float dsel = bd[0]; int isel = bi[0];
  int cnt = 0;
#pragma unroll
  for (int j = 0; j < KNN; ++j) {
    if (j == sub) { dsel = bd[j]; isel = bi[j]; }
    cnt += (bd[j] < r2);  // neighbor_num = (D < r^2).sum(-1) over the k returned (npc.py:262)
  }
  K.D[(size_t)p * KNN + sub] = dsel;
  K.I[(size_t)p * KNN + sub] = isel;
  if (sub == 0) K.nn[p] = cnt;
}

// ---------------------------------------------------------- interpolation ---
struct InterpParams {
  KnnParams K;
  const float* feats; const unsigned char* fmask;
  const float* rand_feat;
  int min_nn;
  float* c;          // [32][P]
  unsigned char* has_nb;  // [P]
  // backward
  const float* dc;   // [32][P]
  float* d_feats;
  float* dp;         // [3][P] accumulated
  int need_dp;
};

__device__ __forceinline__ void nb_weights(const InterpParams& Q, int p, const float q[3],
                                           float w[KNN], float a[KNN], int id[KNN], float& A) {
  const float r = Q.K.radius[p / Q.K.radius_div];
  const float r2 = r * r;
  A = 0.f;
#pragma unroll
  for (int j = 0; j < KNN; ++j) {
    id[j] = Q.K.I[(size_t)p * KNN + j];
    float aj = 0.f;
    if (id[j] >= 0) {
      const float d2 = sqdist(q, Q.K.ix.pos + (size_t)id[j] * 3);  // re-computed (is_tracker path)
      aj = (d2 > r2) ? 0.f : 1.0f / (d2 + 1e-10f);
    }
    a[j] = aj;
    A += fabsf(aj);
  }
  A = fmaxf(A, 1e-12f);  // F.normalize(p=1, eps=1e-12)
#pragma unroll
  for (int j = 0; j < KNN; ++j) w[j] = a[j] / A;
}

__global__ void __launch_bounds__(128) k_interp_fwd(const InterpParams Q) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Q.K.P) return;
  float q[3];
  query_point(Q.K, p, q);
  const bool has = Q.K.nn[p] > Q.min_nn - 1;
  Q.has_nb[p] = has;
  float c[CD];
#pragma unroll
  for (int m = 0; m < CD; ++m) c[m] = 0.f;
  if (has) {
    float w[KNN], a[KNN], A; int id[KNN];
    nb_weights(Q, p, q, w, a, id, A);
#pragma unroll
    for (int j = 0; j < KNN; ++j) {
      if (id[j] < 0 || w[j] == 0.f) continue;
      if (Q.fmask && !Q.fmask[id[j]]) continue;  // geo_feats * frustum_mask
      const float4* f = reinterpret_cast<const float4*>(Q.feats + (size_t)id[j] * CD);
#pragma unroll
      for (int m4 = 0; m4 < CD / 4; ++m4) {
        const float4 v = __ldg(&f[m4]);
        c[4 * m4] = fmaf(w[j], v.x, c[4 * m4]); c[4 * m4 + 1] = fmaf(w[j], v.y, c[4 * m4 + 1]);
        c[4 * m4 + 2] = fmaf(w[j], v.z, c[4 * m4 + 2]); c[4 * m4 + 3] = fmaf(w[j], v.w, c[4 * m4 + 3]);
      }
    }
  } else if (Q.rand_feat) {
#pragma unroll
    for (int m = 0; m < CD; ++m) c[m] = Q.rand_feat[m];
  }
#pragma unroll
  for (int m = 0; m < CD; ++m) Q.c[(size_t)m * Q.K.P + p] = c[m];
}

__global__ void __launch_bounds__(128) k_interp_bwd(const InterpParams Q) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Q.K.P) return;
  if (!Q.has_nb[p]) return;  // constant feature: no gradient
  float q[3];
  query_point(Q.K, p, q);
  float w[KNN], a[KNN], A; int id[KNN];
  nb_weights(Q, p, q, w, a, id, A);
  float dc[CD];
#pragma unroll
  for (int m = 0; m < CD; ++m) dc[m] = Q.dc[(size_t)m * Q.K.P + p];
  float dw[KNN];
  float sw = 0.f;
#pragma unroll
  for (int j = 0; j < KNN; ++j) {
    dw[j] = 0.f;
    if (id[j] < 0 || a[j] == 0.f) continue;
    const bool on = !Q.fmask || Q.fmask[id[j]];
    if (on) {
      const float4* f = reinterpret_cast<const float4*>(Q.feats + (size_t)id[j] * CD);
      float s = 0.f;
#pragma unroll
      for (int m4 = 0; m4 < CD / 4; ++m4) {
        const float4 v = __ldg(&f[m4]);
        s += v.x * dc[4 * m4] + v.y * dc[4 * m4 + 1] + v.z * dc[4 * m4 + 2] + v.w * dc[4 * m4 + 3];
      }
      dw[j] = s;
      if (Q.d_feats)
#pragma unroll
        for (int m4 = 0; m4 < CD / 4; ++m4)
          red_add_v4(Q.d_feats + (size_t)id[j] * CD + 4 * m4, w[j] * dc[4 * m4], w[j] * dc[4 * m4 + 1],
                     w[j] * dc[4 * m4 + 2], w[j] * dc[4 * m4 + 3]);
    }
    sw += w[j] * dw[j];
  }
  if (!Q.need_dp) return;
  // w = a / A (a >= 0): dL/da_j = (dw_j - sum_i w_i dw_i) / A ; a = 1/(D+eps): da/dD = -a^2 ;
  // D = |x - p|^2: dD/dp = -2 (x - p)
  float g[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < KNN; ++j) {
    if (id[j] < 0 || a[j] == 0.f) continue;
    const float da = (dw[j] - sw) / A;
    const float dD = -da * a[j] * a[j];
    const float* x = Q.K.ix.pos + (size_t)id[j] * 3;
#pragma unroll
    for (int d = 0; d < 3; ++d) g[d] += dD * (-2.f) * (x[d] - q[d]);
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) Q.dp[(size_t)d * Q.K.P + p] += g[d];
}

// ------------------------------------------------------------- per ray ---
// torch.linspace(start, end, n)[k] in f32: the two-sided formula of torch's kernel
__device__ __forceinline__ float linspace_f32(float start, float end, int n, int k) {
  const float step = (end - start) / (float)(n - 1);
  return (k < n / 2) ? __fadd_rn(start, __fmul_rn(step, (float)k))
                     : __fsub_rn(end, __fmul_rn(step, (float)(n - 1 - k)));
}

// np.linspace(start, stop, n)[k] in f64 (numpy's function_base.linspace: arange * step + start,
// the step == 0 branch (arange / div) * delta, and the last element set to stop)
__device__ __forceinline__ double linspace_np(double start, double stop, int n, int k) {
  if (k == n - 1) return stop;
  const double div = (double)(n - 1), delta = __dsub_rn(stop, start);
  const double step = __ddiv_rn(delta, div);
  const double y = (step == 0.0) ? __dmul_rn(__ddiv_rn((double)k, div), delta)
                                 : __dmul_rn((double)k, step);
  return __dadd_rn(y, start);
}

// ---------------------------------------------------- samples near the cloud ---
// NeuralPointCloud.sample_near_pcl (neural_point_cloud.py:284-348) for the rays without depth:
// one warp per ray, lane k < 25 tests march point k for a cloud point with D < r^2.
constexpr int NEAR_MARCH = 25;

struct NearP {
  XrdPointIndex ix;
  int R, S;
  const float *rays_o, *rays_d, *target_d, *far;
  double near_end;
  float r_walk, r2;
  float* z;                 // [R][S]
  unsigned char* near;      // [R]
};

__global__ void __launch_bounds__(128) k_near_pcl(const NearP N) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= N.R) return;  // warp-uniform
  if (N.target_d[r] > 0.f) {
    if (lane == 0) N.near[r] = 1;
    return;
  }
  bool hit = false;
  if (lane < NEAR_MARCH && N.ix.n_points > 0) {
    const float zq = linspace_f32((float)N.near_end, N.far[0], NEAR_MARCH, lane);
    float q[3];
#pragma unroll
    for (int d = 0; d < 3; ++d)
      q[d] = __fadd_rn(N.rays_o[r * 3 + d], __fmul_rn(N.rays_d[r * 3 + d], zq));
    walk_cells(N.ix, q, N.r_walk, 0, 1, [&](int, const float* x) {
      hit = sqdist(q, x) < N.r2;
      return hit;
    });
  }
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  const bool valid = __popc(m) >= 2;
  if (lane == 0) N.near[r] = valid;
  if (lane >= N.S) return;
  // first and second hit (the reference's item[0], item[1]), else near_end .. far
  const double far = (double)N.far[0];
  double a = N.near_end, b = far;
  if (valid) {
    const int c0 = __ffs(m) - 1, c1 = __ffs(m & (m - 1)) - 1;
    a = linspace_np(N.near_end, far, NEAR_MARCH, c0);
    b = linspace_np(N.near_end, far, NEAR_MARCH, c1);
  }
  N.z[r * N.S + lane] = __double2float_rn(linspace_np(a, b, N.S, lane));
}

struct RayP {
  int R, S;
  const float *rays_o, *rays_d, *target_s, *target_d;
  const float *t_surface, *far;
  const float* z_near;            // [R][S] samples of the zero-depth rays, or NULL
  const unsigned char* near;      // [R] with z_near: zero-depth ray close to the cloud
  float near_s, far_s, near_end, coef;
  float* z;                       // [R][S]
  const float* occ;               // [P]
  const unsigned char* has_nb;    // [P]
  int min_valid;                  // int(S/2 + 1)
  float *o_rgb, *o_depth, *o_var; unsigned char* o_valid;
  // loss / backward
  int is_mapping, handle_dynamic;
  float* gd;                      // [R] d loss / d depth
  float* tmp;                     // [R]
  float* losses;
  float* d_occ;                   // [P]
  // stage colour
  int stage, Pp, use_color_trk;
  float w_color;
  const float* rgb3;              // [3][Pp] per-sample sigmoid colour
  float* grgb;                    // [R][3] d loss / d rgb_map
  float* d_raw3;                  // [3][Pp] d loss / d (pre-sigmoid colour)
};

__global__ void __launch_bounds__(128) k_sample_z(const RayP P) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P.R) return;
  const float d = P.target_d[r];
  const int S = P.S;
  if (d > 0.f) {
    const float a = __fmul_rn(P.near_s, d), b = __fmul_rn(P.far_s, d);
    for (int k = 0; k < S; ++k) {
      const float t = P.t_surface[k];
      P.z[r * S + k] = __fadd_rn(__fmul_rn(a, __fsub_rn(1.f, t)), __fmul_rn(b, t));
    }
  } else if (P.z_near) {
    for (int k = 0; k < S; ++k) P.z[r * S + k] = P.z_near[r * S + k];
  } else {
    // torch.linspace(near_end, max(far), S): scalar formula (S < SIMD width)
    for (int k = 0; k < S; ++k) P.z[r * S + k] = linspace_f32(P.near_end, P.far[0], S, k);
  }
}

// raw2outputs_nerf_color2 (occupancy, normalised by the weight sum), stage geometry: rgb = 0
__global__ void __launch_bounds__(128) k_composite_fwd(const RayP P) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P.R) return;
  const int S = P.S;
  float T = 1.f, ws = 0.f, nd = 0.f;
  float w[16];
  int nvalid = 0;
  for (int k = 0; k < S; ++k) {
    const int p = r * S + k;
    const bool nb = P.has_nb[p];
    nvalid += nb;
    const float occ = nb ? P.occ[p] : -100.f;
    const float alpha = sigmoidf_acc(P.coef * occ);
    w[k] = alpha * T;
    T *= (1.f - alpha + 1e-10f);
    ws += w[k];
    nd = fmaf(w[k], P.z[p], nd);
  }
  const float wsum = ws + 1e-10f;
  const float depth = nd / wsum;
  float var = 0.f;
  for (int k = 0; k < S; ++k) { const float t = P.z[r * S + k] - depth; var = fmaf(w[k] * t, t, var); }
  const bool nz = P.target_d[r] > 0.f;
  // depth[~gt_non_zero_mask] = 0 unless rendering_sample_near_pcl
  P.o_depth[r] = (nz || P.z_near) ? depth : 0.f;
  P.o_var[r] = var;
  for (int c = 0; c < 3; ++c) {
    float acc = 0.f;
    if (P.stage == 1)
      for (int k = 0; k < S; ++k) acc = fmaf(w[k], P.rgb3[(size_t)c * P.Pp + r * S + k], acc);
    P.o_rgb[r * 3 + c] = acc / wsum;
  }
  P.o_valid[r] = !(nvalid < P.min_valid) && (nz || !P.z_near || P.near[r]);
}

__global__ void __launch_bounds__(1024) k_loss(const RayP P) {
  __shared__ double red[32], redc[32];
  __shared__ float s_med;
  const int tid = threadIdx.x;
  double ld = 0.0, lc = 0.0;
  const bool col = P.is_mapping ? (P.stage == 1) : (P.use_color_trk != 0);
  auto colour = [&](int r, bool m) {  // w_color * sum |target - colour| over the masked rays
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float g = 0.f;
      if (m && col && P.target_s) {
        const float t = P.target_s[r * 3 + c], v = P.o_rgb[r * 3 + c];
        lc += (double)fabsf(t - v);
        g = P.w_color * ((v > t) ? 1.f : ((v < t) ? -1.f : 0.f));
      }
      P.grgb[r * 3 + c] = g;
    }
  };
  if (P.is_mapping) {
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float D = P.target_d[r], d = P.o_depth[r];
      const bool m = (D > 0.f) && P.o_valid[r] && !isnan(d);
      float g = 0.f;
      if (m) { ld += (double)fabsf(D - d); g = (d > D) ? 1.f : ((d < D) ? -1.f : 0.f); }
      P.gd[r] = g;
      colour(r, m);
    }
  } else {
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float e = fabsf(P.target_d[r] - P.o_depth[r]);
      P.tmp[r] = P.handle_dynamic ? e / sqrtf(P.o_var[r] + 1e-10f) : e;
    }
    __syncthreads();
    const int want = (P.R - 1) / 2;
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float v = P.tmp[r];
      int rank = 0;
      for (int j = 0; j < P.R; ++j) { const float u = P.tmp[j]; rank += (u < v) || (u == v && j < r); }
      if (rank == want) s_med = v;
    }
    __syncthreads();
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float D = P.target_d[r], d = P.o_depth[r], var = P.o_var[r];
      const bool m = (P.tmp[r] < 10.f * s_med) && (D > 0.f) && !isnan(d) && !isnan(var);
      float g = 0.f;
      if (m) {
        const float inv = 1.0f / sqrtf(var + 1e-10f);
        const float t = fabsf(D - d) * inv;
        ld += (double)fminf(fmaxf(t, 0.f), 1e3f);
        if (t < 1e3f) g = ((d > D) ? inv : ((d < D) ? -inv : 0.f));
      }
      P.gd[r] = g;
      colour(r, m);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ld += __shfl_xor_sync(0xffffffffu, ld, o);
    lc += __shfl_xor_sync(0xffffffffu, lc, o);
  }
  if ((tid & 31) == 0) { red[tid >> 5] = ld; redc[tid >> 5] = lc; }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[i]; b += redc[i]; }
    P.losses[0] = (float)a;
    P.losses[1] = P.w_color * (float)b;
  }
}

__global__ void __launch_bounds__(128) k_composite_bwd(const RayP P) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P.R) return;
  const int S = P.S;
  const bool nz = P.target_d[r] > 0.f;
  // zero-depth rays: depth overwritten by 0 (no gradient) unless rendering_sample_near_pcl
  const float gd = (nz || P.z_near) ? P.gd[r] : 0.f;
  float alpha[16], Tt[16], w[16];
  float T = 1.f, ws = 0.f, nd = 0.f;
  for (int k = 0; k < S; ++k) {
    const int p = r * S + k;
    const float occ = P.has_nb[p] ? P.occ[p] : -100.f;
    alpha[k] = sigmoidf_acc(P.coef * occ);
    Tt[k] = T;
    w[k] = alpha[k] * T;
    T *= (1.f - alpha[k] + 1e-10f);
    ws += w[k];
    nd = fmaf(w[k], P.z[p], nd);
  }
  const float wsum = ws + 1e-10f, depth = nd / wsum;
  float gc[3] = {0.f, 0.f, 0.f}, cmap[3] = {0.f, 0.f, 0.f};
  if (P.stage == 1)
    for (int c = 0; c < 3; ++c) { gc[c] = P.grgb[r * 3 + c]; cmap[c] = P.o_rgb[r * 3 + c]; }
  // depth = sum w z / wsum, rgb = sum w c / wsum -> dL/dw_k = [gd (z_k - depth) + g.(c_k - rgb)] / wsum
  float suffix = 0.f;
  for (int k = S - 1; k >= 0; --k) {
    const int p = r * S + k;
    float q = gd * (P.z[p] - depth) / wsum;
    if (P.stage == 1)
      for (int c = 0; c < 3; ++c) {
        const float v = P.rgb3[(size_t)c * P.Pp + p];
        q += gc[c] * (v - cmap[c]) / wsum;
        P.d_raw3[(size_t)c * P.Pp + p] = gc[c] * w[k] / wsum * v * (1.f - v);
      }
    const float da = q * Tt[k] - suffix / (1.f - alpha[k] + 1e-10f);
    suffix += q * w[k];
    // raw[~point_mask, -1] = -100 under no_grad: no gradient for samples without neighbours
    P.d_occ[p] = P.has_nb[p] ? da * P.coef * alpha[k] * (1.f - alpha[k]) : 0.f;
  }
}

__global__ void __launch_bounds__(128) k_rayreduce_f(int R, int S, int P, const float* z,
                                                     const float* dp, float* d_o, float* d_d) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float a[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < S; ++k) {
    const size_t p = (size_t)r * S + k;
#pragma unroll
    for (int d = 0; d < 3; ++d) { const float g = dp[(size_t)d * P + p]; a[d] += g; a[3 + d] += g * z[p]; }
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (d_o) d_o[r * 3 + d] = a[d];
    if (d_d) d_d[r * 3 + d] = a[3 + d];
  }
}

#include "pointslam_color.cuh"

}  // namespace point
}  // namespace xrd

using namespace xrd;
using namespace xrd::point;

// ---- index build (SURVEY f2 / VERDICT r01 row 9): counting sort of the point ids by bucket,
// all on the device: histogram -> exclusive scan -> scatter -> per-bucket id sort (the kNN
// result does not depend on the order inside a bucket; sorting makes the index deterministic
// and equal to a stable argsort of the bucket keys).
namespace xrd {
namespace point {
static __global__ void k_ix_hist(const float* pos, int n, float inv_cell, int table, int* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* x = pos + (size_t)i * 3;
  const uint32_t b = bucket_of((int)floorf(x[0] * inv_cell), (int)floorf(x[1] * inv_cell),
                               (int)floorf(x[2] * inv_cell), table);
  atomicAdd(count + b, 1);
}
// single-block exclusive scan over `table` counters (table <= 2^24, power of two): 4096 per
// round (int4 per thread), warp scans + one carry
static __global__ void __launch_bounds__(1024) k_ix_scan(const int* count, int table, int* start, int* end,
                                                          int* cursor) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < table; base += 4096) {
    const int i = base + threadIdx.x * 4;
    int c[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) c[k] = (i + k < table) ? count[i + k] : 0;
    const int mine = c[0] + c[1] + c[2] + c[3];
    int inc = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      int t = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += v;
      }
      warp_tot[lane] = t;  // inclusive over warps
    }
    __syncthreads();
    int before = carry + (warp ? warp_tot[warp - 1] : 0) + inc - mine;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k < table) { start[i + k] = before; end[i + k] = before + c[k]; cursor[i + k] = before; }
      before += c[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_tot[31];
    __syncthreads();
  }
}
static __global__ void k_ix_fill(const float* pos, int n, float inv_cell, int table, int* cursor, int* ids) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* x = pos + (size_t)i * 3;
  const uint32_t b = bucket_of((int)floorf(x[0] * inv_cell), (int)floorf(x[1] * inv_cell),
                               (int)floorf(x[2] * inv_cell), table);
  ids[atomicAdd(cursor + b, 1)] = i;
}
static __global__ void k_ix_sort(int table, const int* start, const int* end, int* ids) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= table) return;
  const int s = start[b], e = end[b];
  for (int i = s + 1; i < e; ++i) {  // insertion sort: buckets hold a handful of points
    const int v = ids[i];
    int j = i - 1;
    while (j >= s && ids[j] > v) { ids[j + 1] = ids[j]; --j; }
    ids[j + 1] = v;
  }
}
}  // namespace point
}  // namespace xrd

struct KnnWs : Carver {
  KnnWs(void* base, int table_size)
      : Carver(base), count(take<int>((size_t)table_size)), cursor(take<int>((size_t)table_size)) {}
  int *count, *cursor;
};

extern "C" size_t xrd_pointslam_knn_build_workspace_bytes(int table_size) {
  return KnnWs(nullptr, table_size).bytes();
}

extern "C" int xrd_pointslam_knn_build(const float* pos, int n_points, float cell, int table_size,
                                       int32_t* cell_start, int32_t* cell_end, int32_t* sorted_ids,
                                       void* workspace, size_t workspace_bytes, void* stream_) {
  if (!cell_start || !cell_end || !workspace) return XRD_E_NULL;
  if (n_points > 0 && (!pos || !sorted_ids)) return XRD_E_NULL;
  if (table_size < 1 || table_size > (1 << 24) || (table_size & (table_size - 1)) || !(cell > 0.f))
    return XRD_E_SHAPE;
  const KnnWs L(workspace, table_size);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  int *count = L.count, *cursor = L.cursor;
  const float inv = (1.0f / cell);
  XRD_CUDA_TRY(cudaMemsetAsync(count, 0, (size_t)table_size * sizeof(int), stream));
  if (n_points > 0) {
    point::k_ix_hist<<<(n_points + 255) / 256, 256, 0, stream>>>(pos, n_points, inv, table_size, count);
    XRD_LAUNCH_CHECK();
  }
  point::k_ix_scan<<<1, 1024, 0, stream>>>(count, table_size, cell_start, cell_end, cursor);
  XRD_LAUNCH_CHECK();
  if (n_points > 0) {
    point::k_ix_fill<<<(n_points + 255) / 256, 256, 0, stream>>>(pos, n_points, inv, table_size, cursor,
                                                                 sorted_ids);
    XRD_LAUNCH_CHECK();
    point::k_ix_sort<<<(table_size + 255) / 256, 256, 0, stream>>>(table_size, cell_start, cell_end,
                                                                   sorted_ids);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}

extern "C" int xrd_pointslam_knn_query(const XrdPointIndex* index, const float* queries,
                                       const float* radius, int radius_stride, int n_queries,
                                       float* D, int32_t* I, int32_t* neighbor_num, void* stream) {
  if (!index || !queries || !radius || !D || !I || !neighbor_num) return XRD_E_NULL;
  if (!index->pos || !index->cell_start || !index->cell_end || !index->sorted_ids) return XRD_E_NULL;
  if (index->table_size < 1 || (index->table_size & (index->table_size - 1)) || !(index->cell > 0.f))
    return XRD_E_SHAPE;
  if (n_queries <= 0) return XRD_OK;
  KnnParams K;
  K.ix = *index; K.q = queries; K.rays_o = K.rays_d = K.z = nullptr; K.S = 1;
  K.radius = radius; K.radius_div = radius_stride > 0 ? radius_stride : 1 << 30;
  K.P = n_queries; K.D = D; K.I = I; K.nn = neighbor_num;
  k_knn<<<(int)(((long long)n_queries * KG + 127) / 128), 128, 0, (cudaStream_t)stream>>>(K);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_pointslam_sample_near_pcl(const XrdPointIndex* index, const float* rays_o,
                                             const float* rays_d, const float* target_d,
                                             int n_rays, const float* far, double near_end,
                                             double radius_query, int n_surface, float* z,
                                             uint8_t* near, void* stream) {
  if (!index || !rays_o || !rays_d || !target_d || !far || !z || !near) return XRD_E_NULL;
  if (!index->cell_start || !index->cell_end || !index->sorted_ids) return XRD_E_NULL;
  if (index->n_points > 0 && !index->pos) return XRD_E_NULL;
  if (index->n_points < 0 || index->table_size < 1 || (index->table_size & (index->table_size - 1)) ||
      !(index->cell > 0.f) || !(radius_query >= 0.0))
    return XRD_E_SHAPE;
  if (n_rays <= 0) return XRD_OK;
  if (n_surface < 2 || n_surface > 16) return XRD_E_SHAPE;
  NearP N;
  N.ix = *index; N.R = n_rays; N.S = n_surface;
  N.rays_o = rays_o; N.rays_d = rays_d; N.target_d = target_d; N.far = far;
  N.near_end = near_end;
  // D < radius_query**2: torch compares the f32 distances with the f64 square rounded to f32;
  // the cell box is widened by 1e-4 so that rounding cannot drop a cell holding such a point
  N.r2 = (float)(radius_query * radius_query);
  N.r_walk = (float)radius_query * 1.0001f;
  N.z = z; N.near = near;
  k_near_pcl<<<(int)(((long long)n_rays * 32 + 127) / 128), 128, 0, (cudaStream_t)stream>>>(N);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

namespace {
struct PWs : Carver {
  PWs(void* base, int R, int S, int stage, int with_grads)
      : Carver(base), R(R), P((size_t)R * S), g(with_grads != 0), col(stage == 1) {}
  const size_t R, P, Pp_ = (P + 3) / 4 * 4, Np = 8 * Pp_;
  const bool g, col;
  const int Pp = (int)Pp_;
  float *z = take<float>(P), *D = take<float>(P * KNN);
  int *I = take<int>(P * KNN), *nn = take<int>(P);
  float* c = take<float>(CD * P);
  unsigned char* has = take<unsigned char>(P);
  float* occ = take<float>(P);
  // with_grads only
  float *d_occ = g ? take<float>(P) : nullptr, *dc = g ? take<float>(CD * P) : nullptr;
  float *dp = g ? take<float>(3 * P) : nullptr, *gd = g ? take<float>(R) : nullptr;
  float* tmp = g ? take<float>(R) : nullptr;
  uint32_t* masks = g ? take<uint32_t>(5 * P) : nullptr;
  float* grgb = g ? take<float>(R * 3) : nullptr;
  // stage colour ([rows][Pp] / [rows][8 Pp] float arrays)
  float* wn = col ? take<float>(8 * Pp_) : nullptr;
  float *Xn = rows(CNI, Np), *Hn = rows(CW, Np), *Fn = rows(CD, Np), *cc = rows(CD, Pp_);
  float *X3 = rows(CX3, Pp_), *act = rows(5 * CW, Pp_), *H = rows(4 * CW, Pp_), *T = rows(CW, Pp_);
  float* rgb3 = rows(3, Pp_);
  // stage colour with_grads only
  float *d_raw3 = grows(3, Pp_), *g0 = grows(CW, Pp_), *g1 = grows(CW, Pp_), *gp = grows(CW, Pp_);
  float *dX3 = grows(CX3, Pp_), *dcc = grows(CD, Pp_), *dFn = grows(CD, Np), *dHn = grows(CW, Np);
  float* dXn = grows(CNI, Np);

 private:
  float* rows(size_t n, size_t w) { return col ? take<float>(n * w) : nullptr; }
  float* grows(size_t n, size_t w) { return col && g ? take<float>(n * w) : nullptr; }
};

#define XRD_GEMM(...)                                         \
  do {                                                        \
    GemmArgs g_ = __VA_ARGS__;                                \
    XRD_CUDA_TRY(launch_gemm(g_, stream));                    \
  } while (0)

// ---- stage colour: forward -----------------------------------------------------------------
int color_forward(const ColorP& C0, const PWs& L, int P, cudaStream_t stream) {
  const XrdPointColorDecoder& d = C0.dec;
  const int Pp = L.Pp, Np = 8 * Pp;
  float *Xn = L.Xn, *Hn = L.Hn, *Fn = L.Fn, *cc = L.cc, *X3 = L.X3, *T = L.T;
  // only the first P of every Pp-wide slot holds data; the neighbour GEMMs (and their weight
  // gradients) run over the padded width: pad columns must be zero
  if (Pp != P) XRD_CUDA_TRY(cudaMemsetAsync(Xn, 0, (size_t)CNI * Np * sizeof(float), stream));
  k_nb_build<<<(P + 127) / 128, 128, 0, stream>>>(C0);
  XRD_LAUNCH_CHECK();
  XRD_GEMM({CW, Np, CNI, d.nb_w1, CNI, 0, Xn, Np, Hn, Np, d.nb_b1, ACT_SOFTPLUS100, nullptr, 0, nullptr, 0, 0});
  XRD_GEMM({CD, Np, CW, d.nb_w2, CW, 0, Hn, Np, Fn, Np, d.nb_b2, ACT_NONE, nullptr, 0, nullptr, 0, 0});
  k_nb_reduce<<<(P + 127) / 128, 128, 0, stream>>>(C0);
  XRD_LAUNCH_CHECK();
  // trunk: inputs  emb(40) | H0 | H1 | X3 = [emb, H2](168) | H3 ; outputs H0 H1 H2(in X3) H3 H4
  float* Hs[5] = {L.H, L.H + (size_t)CW * Pp, X3 + (size_t)2 * CE * Pp,
                  L.H + (size_t)2 * CW * Pp, L.H + (size_t)3 * CW * Pp};
  const float* in[5] = {X3, Hs[0], Hs[1], X3, Hs[3]};
  const int kin[5] = {2 * CE, CW, CW, CX3, CW};
  for (int i = 0; i < 5; ++i) {
    XRD_GEMM({CW, P, CD, d.wc[i], CD, 0, cc, Pp, T, Pp, d.bc[i], ACT_NONE, nullptr, 0, nullptr, 0, 0});
    XRD_GEMM({CW, P, kin[i], d.w[i], kin[i], 0, in[i], Pp, Hs[i], Pp, d.b[i], ACT_SOFTPLUS100, T, Pp,
              L.act + (size_t)i * CW * Pp, Pp, 0});
  }
  XRD_GEMM({3, P, CW, d.wo, CW, 0, Hs[4], Pp, L.rgb3, Pp, d.bo, ACT_SIGMOID, nullptr, 0, nullptr, 0, 0});
  return XRD_OK;
}

// ---- stage colour: backward (d_raw3 -> decoder grads, d col_feats, d p) ----------------------
int color_backward(ColorP C, const PWs& L, int P, const XrdPointColorDecoderGrads* G,
                   cudaStream_t stream) {
  const XrdPointColorDecoder& d = C.dec;
  const int Pp = L.Pp, Np = 8 * Pp;
  float *Xn = L.Xn, *Hn = L.Hn, *cc = L.cc, *X3 = L.X3;
  float *g0 = L.g0, *g1 = L.g1, *gp = L.gp, *dX3 = L.dX3, *dcc = L.dcc;
  float *dFn = L.dFn, *dHn = L.dHn, *dXn = L.dXn, *d_raw3 = L.d_raw3;
  float* Hs[5] = {L.H, L.H + (size_t)CW * Pp, X3 + (size_t)2 * CE * Pp,
                  L.H + (size_t)2 * CW * Pp, L.H + (size_t)3 * CW * Pp};
  const float* in[5] = {X3, Hs[0], Hs[1], X3, Hs[3]};
  const int kin[5] = {2 * CE, CW, CW, CX3, CW};
  DwParams Dw;
  auto dw_begin = [&](int cols, int ld) { Dw.n_jobs = 0; Dw.P = cols; Dw.Pp = ld; Dw.chunk = 1024; };
  auto dw_add = [&](const float* a, int nA, const float* b, int nB, float* o, int ldo, float* bias) {
    // out[j][i] += sum_p b_j[p] a_i[p], rows of b in groups of 32
    if (!o && !bias) return;
    for (int c = 0; c < nB; c += 32) {
      DwJob& J = Dw.jobs[Dw.n_jobs++];
      J.A = a; J.nA = o ? nA : 0; J.B = b + (size_t)c * Dw.Pp; J.nB = nB - c < 32 ? nB - c : 32;
      J.mask = nullptr; J.out = o ? o + (size_t)c * ldo : nullptr; J.sj = ldo; J.si = 1;
      J.bias = bias ? bias + c : nullptr;
    }
  };
  auto dw_run = [&]() -> int {
    if (Dw.n_jobs == 0) return XRD_OK;
    if (Dw.n_jobs > DW_MAX_JOBS) return XRD_E_SHAPE;
    XRD_CUDA_TRY(launch_dw(Dw, stream));
    return XRD_OK;
  };
  int st;
  // output layer
  XRD_GEMM({CW, P, 3, d.wo, CW, 1, d_raw3, Pp, g0, Pp, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, 0});
  if (G) {
    dw_begin(P, Pp);
    dw_add(Hs[4], CW, d_raw3, 3, G->wo, CW, G->bo);
    if ((st = dw_run()) != XRD_OK) return st;
  }
  float* dH[5] = {g1, g0, dX3 + (size_t)2 * CE * Pp, g1, g0};  // where dH_i lives
  float* dIn[5] = {dX3, g1, g0, dX3, g1};                       // where W_i^T dPre_i goes
  for (int i = 4; i >= 0; --i) {
    // fc_c branch: dc += wc_i^T dH_i
    XRD_GEMM({CD, P, CW, d.wc[i], CD, 1, dH[i], Pp, dcc, Pp, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, i == 4 ? 0 : 1});
    const size_t n = (size_t)CW * Pp;
    k_dsoftplus<<<592, 256, 0, stream>>>(n, dH[i], L.act + (size_t)i * CW * Pp, gp);
    XRD_LAUNCH_CHECK();
    if (G) {
      dw_begin(P, Pp);
      dw_add(cc, CD, dH[i], CW, G->wc[i], CD, G->bc[i]);
      dw_add(in[i], kin[i], gp, CW, G->w[i], kin[i], G->b[i]);
      if ((st = dw_run()) != XRD_OK) return st;
    }
    if (i > 0) {
      XRD_GEMM({kin[i], P, CW, d.w[i], kin[i], 1, gp, Pp, dIn[i], Pp, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, 0});
    } else if (C.need_dp) {  // layer 0: d embedding accumulates onto block 3's share
      XRD_GEMM({kin[0], P, CW, d.w[0], kin[0], 1, gp, Pp, dX3, Pp, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, 1});
    }
  }
  // neighbour MLP
  C.dcc = dcc; C.dFn = dFn; C.dXn = dXn; C.dX3 = dX3;
  C.d_B_rel = G ? G->B_rel : nullptr;
  if (Pp != P) XRD_CUDA_TRY(cudaMemsetAsync(dFn, 0, (size_t)CD * Np * sizeof(float), stream));
  k_nb_reduce_bwd<<<(P + 127) / 128, 128, 0, stream>>>(C);
  XRD_LAUNCH_CHECK();
  XRD_GEMM({CW, Np, CD, d.nb_w2, CW, 1, dFn, Np, dHn, Np, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, 0});
  k_dsoftplus<<<1184, 256, 0, stream>>>((size_t)CW * Np, dHn, Hn, dHn);
  XRD_LAUNCH_CHECK();
  if (G) {
    dw_begin(Np, Np);
    dw_add(Hn, CW, dFn, CD, G->nb_w2, CW, G->nb_b2);
    dw_add(Xn, CNI, dHn, CW, G->nb_w1, CNI, G->nb_b1);
    if ((st = dw_run()) != XRD_OK) return st;
  }
  XRD_GEMM({CNI, Np, CW, d.nb_w1, CNI, 1, dHn, Np, dXn, Np, nullptr, ACT_NONE, nullptr, 0, nullptr, 0, 0});
  k_nb_build_bwd<<<(P + 127) / 128, 128, 0, stream>>>(C);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
}  // namespace

extern "C" size_t xrd_pointslam_workspace_bytes(int n_rays, int n_surface, int stage, int with_grads) {
  return PWs(nullptr, n_rays, n_surface, stage, with_grads).bytes();
}

extern "C" int xrd_pointslam_step(const XrdRays* rays, const XrdPointIndex* index,
                                  const XrdPointFeats* feats, const XrdNiceDecoder* dec,
                                  const XrdPointColorDecoder* cdec, const XrdPointCfg* cfg,
                                  XrdPointOut* out, XrdPointGrads* grads,
                                  void* workspace, size_t workspace_bytes, void* stream_) {
  if (!rays || !index || !feats || !dec || !cfg || !out || !workspace) return XRD_E_NULL;
  if (!rays->rays_o || !rays->rays_d || !rays->target_d || !feats->geo_feats) return XRD_E_NULL;
  if (!cfg->t_surface || !cfg->far || !cfg->radius_query) return XRD_E_NULL;
  if (!cfg->near_pcl_z != !cfg->near_pcl_mask) return XRD_E_NULL;
  if (!out->rgb || !out->depth || !out->uncertainty || !out->valid_ray_mask) return XRD_E_NULL;
  const int stage = cfg->stage;
  if (stage != 0 && stage != 1) return XRD_E_SHAPE;
  if (stage == 1) {
    if (!cdec || !feats->col_feats) return XRD_E_NULL;
    const float* const* arrs[4] = {cdec->w, cdec->b, cdec->wc, cdec->bc};
    for (auto a : arrs) for (int i = 0; i < 5; ++i) if (!a[i]) return XRD_E_NULL;
    if (!cdec->B || !cdec->B_rel || !cdec->nb_w1 || !cdec->nb_b1 || !cdec->nb_w2 || !cdec->nb_b2 ||
        !cdec->wo || !cdec->bo)
      return XRD_E_NULL;
    if (grads && !rays->target_s) return XRD_E_NULL;
    if (grads && grads->color) {  // colour-decoder gradients are all-or-nothing
      const XrdPointColorDecoderGrads* G = grads->color;
      float* const* ga[4] = {G->w, G->b, G->wc, G->bc};
      for (auto a : ga) for (int i = 0; i < 5; ++i) if (!a[i]) return XRD_E_NULL;
      if (!G->B_rel || !G->nb_w1 || !G->nb_b1 || !G->nb_w2 || !G->nb_b2 || !G->wo || !G->bo)
        return XRD_E_NULL;
    }
  }
  if (dec->c_dim != CD || dec->n_out != 1) return XRD_E_SHAPE;
  const int R = rays->n_rays, S = cfg->n_surface;
  if (R <= 0) return XRD_OK;
  if (S < 2 || S > 16) return XRD_E_SHAPE;
  if (grads && !out->losses) return XRD_E_NULL;
  if (grads && !cfg->is_mapping && R > 8192) return XRD_E_SHAPE;
  const PWs L(workspace, R, S, stage, grads != nullptr);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = R * S;
  float* z = out->z_vals ? out->z_vals : L.z;

  RayP Y;
  Y.R = R; Y.S = S; Y.rays_o = rays->rays_o; Y.rays_d = rays->rays_d;
  Y.target_s = rays->target_s; Y.target_d = rays->target_d; Y.t_surface = cfg->t_surface;
  Y.far = cfg->far; Y.near_s = cfg->near_end_surface; Y.far_s = cfg->far_end_surface;
  Y.z_near = cfg->near_pcl_z; Y.near = cfg->near_pcl_mask;
  Y.near_end = cfg->near_end; Y.coef = cfg->sigmoid_coef; Y.z = z;
  Y.occ = L.occ;
  Y.has_nb = L.has;
  Y.min_valid = S / 2 + 1;
  Y.o_rgb = out->rgb; Y.o_depth = out->depth; Y.o_var = out->uncertainty; Y.o_valid = out->valid_ray_mask;
  Y.is_mapping = cfg->is_mapping; Y.handle_dynamic = cfg->handle_dynamic;
  Y.gd = nullptr; Y.tmp = nullptr; Y.losses = out->losses; Y.d_occ = nullptr;
  Y.stage = stage; Y.Pp = L.Pp; Y.use_color_trk = cfg->use_color_in_tracking; Y.w_color = cfg->w_color;
  Y.rgb3 = L.rgb3;
  Y.grgb = nullptr; Y.d_raw3 = nullptr;
  k_sample_z<<<(R + 127) / 128, 128, 0, stream>>>(Y);
  XRD_LAUNCH_CHECK();

  InterpParams Q;
  Q.K.ix = *index; Q.K.q = nullptr; Q.K.rays_o = rays->rays_o; Q.K.rays_d = rays->rays_d; Q.K.z = z;
  Q.K.S = S; Q.K.radius = cfg->radius_query; Q.K.radius_div = S; Q.K.P = P;
  Q.K.D = L.D; Q.K.I = L.I;
  Q.K.nn = L.nn;
  Q.feats = feats->geo_feats; Q.fmask = feats->frustum_mask; Q.rand_feat = cfg->rand_feat;
  Q.min_nn = cfg->min_nn_num; Q.c = L.c;
  Q.has_nb = L.has;
  Q.dc = nullptr; Q.d_feats = nullptr; Q.dp = nullptr; Q.need_dp = 0;
  {
    KernelTimer kt(stream);
    k_knn<<<(int)(((long long)P * KG + 127) / 128), 128, 0, stream>>>(Q.K);
  }
  XRD_LAUNCH_CHECK();
  k_interp_fwd<<<(P + 127) / 128, 128, 0, stream>>>(Q);
  XRD_LAUNCH_CHECK();

  xrd::nice::DecParams D;
  D.P = P; D.S = S; D.zf = z; D.rays_o = rays->rays_o; D.rays_d = rays->rays_d;
  D.dec = *dec;
  D.out[0] = L.occ;
  D.masks = L.masks;
  D.dp = L.dp;
  D.need_dp = grads && (grads->d_rays_o || grads->d_rays_d);
  D.ext_c = Q.c; D.ext_dc = L.dc;
  D.embed_scale = 6.283185307179586f;  // 2 * math.pi, float32
  XRD_CUDA_TRY(xrd::nice::launch_decoder(D, false, stream));
  ColorP C{};
  if (stage == 1) {
    C.K = Q.K; C.Pp = L.Pp; C.min_nn = cfg->min_nn_num; C.col_feats = feats->col_feats;
    C.rand_feat = cfg->rand_feat_color; C.dec = *cdec;
    C.wn = L.wn; C.Xn = L.Xn;
    C.Fn = L.Fn; C.cc = L.cc;
    C.X3 = L.X3; C.has_nb = Q.has_nb;
    const int st = color_forward(C, L, P, stream);
    if (st != XRD_OK) return st;
  }
  k_composite_fwd<<<(R + 127) / 128, 128, 0, stream>>>(Y);
  XRD_LAUNCH_CHECK();
  if (!grads) return XRD_OK;

  Y.gd = L.gd; Y.tmp = L.tmp;
  Y.d_occ = L.d_occ;
  Y.grgb = L.grgb;
  Y.d_raw3 = L.d_raw3;
  point::k_loss<<<1, 1024, 0, stream>>>(Y);
  XRD_LAUNCH_CHECK();
  k_composite_bwd<<<(R + 127) / 128, 128, 0, stream>>>(Y);
  XRD_LAUNCH_CHECK();
  XRD_CUDA_TRY(cudaMemsetAsync(L.dp, 0, 3 * (size_t)P * 4, stream));
  D.dout[0] = Y.d_occ;
  XRD_CUDA_TRY(xrd::nice::launch_decoder(D, true, stream));
  Q.dc = D.ext_dc; Q.d_feats = grads->d_geo_feats; Q.dp = D.dp; Q.need_dp = D.need_dp;
  k_interp_bwd<<<(P + 127) / 128, 128, 0, stream>>>(Q);
  XRD_LAUNCH_CHECK();
  if (stage == 1) {
    C.dp = D.dp; C.need_dp = D.need_dp; C.d_col_feats = grads->d_col_feats;
    const int st = color_backward(C, L, P, grads->color, stream);
    if (st != XRD_OK) return st;
  }
  if (D.need_dp) {
    k_rayreduce_f<<<(R + 127) / 128, 128, 0, stream>>>(R, S, P, z, D.dp, grads->d_rays_o, grads->d_rays_d);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}
