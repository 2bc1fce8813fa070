// NICE-SLAM render-and-optimise step (sm_90a).
//
// Replaces (reference @ f0366f20): slam/models/conv_onet.py:377-524 render_batch_ray,
// :339-375 eval_points, slam/model_components/decoder_nice.py:386-414 NICE.forward with the
// MLP decoders :207-234 (grid_sample trilerp :195-205, Gaussian Fourier embedding :11-38),
// slam/model_components/utils.py:189-244 raw2outputs_nerf_color, conv_onet.py:145-185
// get_loss_dict and the autograd backward of the chain.
//
// Pipeline of one xrd_nice_step (all on the caller's stream):
//   k_maxdepth      batch-global max(target_d) (far clamp / zero-depth sampling, Q9)
//   k_sample        warp per ray: far from the bound (f64), 32 uniform + 16 surface samples
//                   in f64, the uniform ones jittered when rendering_perturb > 0, rank sort
//                   (== torch.sort values)
//   [n_importance > 0: pass 1 = k_decoder_fwd and k_composite (weights only) over those
//    samples, then k_sample_pdf: sample_pdf on pass 1's weights and the sorted merge; the
//    pipeline below is pass 2, over the merged samples]
//   k_decoder_fwd   x3 (middle [, fine [, color]]): thread per point, 8-lane cooperative
//                   trilerp on the channel-last grid (one voxel = one 128 B line), decoder
//                   weights transposed in shared memory, Fourier embedding + grid feature in
//                   a per-thread shared-memory column, hidden state in registers; relu masks
//                   (and, for the trainable colour decoder, layer inputs) go to an HBM
//                   workspace in [feature][point] order
//   k_composite_fwd warp per ray: occupancy compositing (f32 weights, f64 depth), S <= 64 in
//                   two slots per lane, S <= 128 in four
//   k_loss          per-ray loss coefficients; tracking: batch median of |d-D|/sqrt(var)
//   k_composite_bwd d loss / d occupancy logit, d loss / d rgb per sample
//   k_decoder_bwd   x3: transposed chain with the stored masks, grid scatter
//                   (red.global.add.v4.f32 per 4 channels), coordinate gradients through
//                   trilerp and sin(pB)
//   k_dw            colour-decoder weight gradients: shared-memory tiled X^T dY over points
//   k_rayreduce     d loss / d rays_o, d rays_d
#include <math.h>

#include "mlp.cuh"
#include "nice.cuh"
#include "sample_pdf.cuh"

namespace xrd {
namespace nice {

constexpr int E = 93;    // Fourier embedding size
constexpr int H = 32;    // hidden width
constexpr int T = 192;   // threads per CTA of the decoder kernels
constexpr int CMAX = 64; // fine decoder: own 32 ++ middle 32

// transposed weight block in shared memory (floats)
struct WOff {
  int pts[5];   // [in][32]
  int fcc[5];   // [c_dim][32]
  int out;      // [32][4]
  int B;        // [3][93]
  int pts_b, fcc_b, out_b;
  int total;
};
__host__ __device__ inline WOff woff(int c_dim) {
  WOff o;
  int q = 0;
  const int in[5] = {E, H, H, E + H, H};
  for (int i = 0; i < 5; ++i) { o.pts[i] = q; q += in[i] * H; }
  for (int i = 0; i < 5; ++i) { o.fcc[i] = q; q += c_dim * H; }
  o.out = q; q += H * 4;
  o.B = q; q += 3 * E; q = (q + 3) & ~3;
  o.pts_b = q; q += 5 * H;
  o.fcc_b = q; q += 5 * H;
  o.out_b = q; q += 4;
  o.total = q;
  return o;
}

// rows of the activation workspace (trainable decoder)
__host__ __device__ inline int row_e() { return 0; }
__host__ __device__ inline int row_h(int i) { return E + i * H; }
__host__ __device__ inline int row_c() { return E + 5 * H; }
__host__ __device__ inline int row_dh(int i, int c_dim) { return E + 5 * H + c_dim + i * H; }
__host__ __device__ inline int row_gm(int c_dim) { return E + 5 * H + c_dim + 5 * H; }
__host__ __device__ inline int row_pf(int c_dim) { return row_gm(c_dim) + E; }
__host__ __device__ inline int row_do(int c_dim) { return row_pf(c_dim) + 3; }
__host__ __device__ inline int n_rows(int c_dim) { return row_do(c_dim) + 4; }

// ------------------------------------------------------------- sampling ---
static __global__ void k_maxdepth(const float* d, int R, float* out) {
  __shared__ float sm[32];
  float m = -INFINITY;
  for (int i = threadIdx.x; i < R; i += blockDim.x) m = fmaxf(m, d[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : -INFINITY;
    m = warp_max(m);
    if (threadIdx.x == 0) out[0] = m;
  }
}

struct SampleParams {
  int R, ns, nsurf;
  int no_depth;  // stage 'coarse': gt_depth = None -> near = 0.01, far = far_bb, no surface samples
  const float *rays_o, *rays_d, *target_d;
  double bmin[3], bmax[3];
  const float *t_uniform, *t_surface;  // torch.linspace(0,1,n) tables
  const float* maxd;   // device scalar
  double* z;           // [R][ns+nsurf]
  // PERTURB (rendering_perturb > 0): uniforms of the jitter, [R][ns] or NULL -> Philox(seed)
  const float* noise;
  uint64_t seed;
};

template <bool PERTURB>
static __global__ void __launch_bounds__(128) k_sample(SampleParams p) {
  __shared__ double zs[4][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + warp;
  if (r >= p.R) return;
  const int S = p.ns + p.nsurf;
  double* z = zs[warp];
  const float maxd = p.no_depth ? 0.f : p.maxd[0];
  const float gt = p.no_depth ? 0.f : p.target_d[r];
  // far_bb = min_d max_side (bound - o) / d  (+0.01), all in f64 (conv_onet.py:407-414)
  double far_bb = INFINITY;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double o = (double)p.rays_o[r * 3 + d], dd = (double)p.rays_d[r * 3 + d];
    const double t0 = (p.bmin[d] - o) / dd, t1 = (p.bmax[d] - o) / dd;
    far_bb = fmin(far_bb, fmax(t0, t1));
  }
  far_bb += 0.01;
  const float cap = __fmul_rn(maxd, 1.2f);  // torch.max(gt_depth * 1.2): f32
  const double far = p.no_depth ? far_bb : fmin(fmax(far_bb, 0.0), (double)cap);
  const float near = p.no_depth ? 0.01f : __fmul_rn(gt, 0.01f);
  for (int k = lane; k < S; k += 32) {
    double v;
    if (k < p.ns) {
      // t = linspace(0,1,ns) f32;  near*(1-t) in f32, far*t in f64
      const float t = p.t_uniform[k];
      v = __dadd_rn((double)__fmul_rn(near, __fsub_rn(1.0f, t)), __dmul_rn(far, (double)t));
    } else {
      const int j = k - p.ns;
      const double t = (double)p.t_surface[j];
      // no fma contraction: torch rounds each product before the sum
      if (gt > 0.f)
        v = __dadd_rn(__dmul_rn((double)__fmul_rn(0.95f, gt), 1.0 - t),
                      __dmul_rn((double)__fmul_rn(1.05f, gt), t));
      else
        v = __dadd_rn(__dmul_rn(0.001, 1.0 - t), __dmul_rn((double)maxd, t));
    }
    z[k] = v;
  }
  __syncwarp();
  if (PERTURB) {
    // conv_onet.py:470-477: mids = .5 (z[1:] + z[:-1]), upper = [mids, z[-1]], lower = [z[0],
    // mids], z = lower + (upper - lower) u over the ns uniform samples only, all in f64 with u
    // promoted from f32; each product and sum rounded on its own (no fma contraction)
    double zj[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = lane + 32 * i;
      if (k >= p.ns) break;
      const double lo = k == 0 ? z[0] : __dmul_rn(0.5, __dadd_rn(z[k], z[k - 1]));
      const double hi = k == p.ns - 1 ? z[k] : __dmul_rn(0.5, __dadd_rn(z[k + 1], z[k]));
      float u;
      if (p.noise) {
        u = p.noise[(size_t)r * p.ns + k];
      } else {
        float q[4];
        philox4(p.seed, (uint64_t)r * p.ns + k, q);
        u = q[0];
      }
      zj[i] = __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), (double)u));
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (lane + 32 * i < p.ns) z[lane + 32 * i] = zj[i];
    __syncwarp();
  }
  // rank sort (values equal torch.sort's)
  for (int k = lane; k < S; k += 32) {
    const double v = z[k];
    int rank = 0;
    for (int j = 0; j < S; ++j) {
      const double u = z[j];
      rank += (u < v) || (u == v && j < k);
    }
    p.z[(size_t)r * S + rank] = v;
  }
}

// --------------------------------------------------------------- trilerp ---
// F.grid_sample(align_corners=True, padding_mode='border', bilinear) source index
struct Cell {
  int ix, iy, iz;     // top-north-west corner
  float fx, fy, fz;   // fractional offsets
  float mx, my, mz;   // d(index)/d(normalised coord) incl. border clip (0 when clipped)
};
__device__ __forceinline__ void src_index(float x, int size, int& i0, float& f, float& mult) {
  float ix = ((x + 1.f) / 2.f) * (float)(size - 1);
  mult = (float)(size - 1) / 2.f;
  const float hi = (float)(size - 1);
  // clip_coordinates_set_grad: the coordinate gradient is 0 on the faces too (ix == 0, hi)
  if (ix <= 0.f) { mult = 0.f; ix = fmaxf(ix, 0.f); }
  if (ix >= hi) { mult = 0.f; ix = fminf(ix, hi); }
  const float fl = floorf(ix);
  i0 = (int)fl;
  f = ix - fl;
}

__device__ __forceinline__ void point_f64(const DecParams& P, int p, double pt[3]) {
  const int r = p / P.S;
  if (!P.z) {  // Point-SLAM: pts = rays_o + rays_d * z, all float32
    const float z = P.zf[p];
#pragma unroll
    for (int d = 0; d < 3; ++d)
      pt[d] = (double)__fadd_rn(P.rays_o[r * 3 + d], __fmul_rn(P.rays_d[r * 3 + d], z));
    return;
  }
  const double z = P.z[p];
#pragma unroll
  for (int d = 0; d < 3; ++d)
    pt[d] = __dadd_rn((double)P.rays_o[r * 3 + d], __dmul_rn((double)P.rays_d[r * 3 + d], z));
}

__device__ __forceinline__ Cell make_cell(const DecParams& P, const Grid& g, const double pt[3]) {
  Cell c;
  float xn[3];
#pragma unroll
  for (int d = 0; d < 3; ++d)
    xn[d] = (float)(((pt[d] - P.bmin[d]) / (P.bmax[d] - P.bmin[d])) * 2.0 - 1.0);
  src_index(xn[0], g.nx, c.ix, c.fx, c.mx);
  src_index(xn[1], g.ny, c.iy, c.fy, c.my);
  src_index(xn[2], g.nz, c.iz, c.fz, c.mz);
  return c;
}

// 8 lanes per point (4 channels each), 4 points per warp pass.  The owner lane's cell is
// broadcast with shuffles; the gathered feature lands in the owner's shared-memory column.
__device__ __forceinline__ void trilerp_coop(const Grid& g, const Cell& mine, bool active,
                                             float* __restrict__ ccol0, int tbase) {
  const int lane = threadIdx.x & 31, sub = lane & 7, q = lane >> 3;
#pragma unroll 1
  for (int grp = 0; grp < 8; ++grp) {
    const int owner = grp * 4 + q;
    const int ix = __shfl_sync(0xffffffffu, mine.ix, owner);
    const int iy = __shfl_sync(0xffffffffu, mine.iy, owner);
    const int iz = __shfl_sync(0xffffffffu, mine.iz, owner);
    const float fx = __shfl_sync(0xffffffffu, mine.fx, owner);
    const float fy = __shfl_sync(0xffffffffu, mine.fy, owner);
    const float fz = __shfl_sync(0xffffffffu, mine.fz, owner);
    const int act = __shfl_sync(0xffffffffu, (int)active, owner);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (act) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
        const int x = ix + dx, y = iy + dy, z = iz + dz;
        if (x < g.nx && y < g.ny && z < g.nz) {  // within_bounds_3d (lower bound holds after clip)
          const float w = (dx ? fx : 1.f - fx) * (dy ? fy : 1.f - fy) * (dz ? fz : 1.f - fz);
          const float4 v = __ldg(reinterpret_cast<const float4*>(
              g.data + ((size_t)((size_t)z * g.ny + y) * g.nx + x) * 32 + sub * 4));
          acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
          acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
        }
      }
    }
    float* col = ccol0 + (tbase + owner);  // column of the owner thread
    col[(sub * 4 + 0) * T] = acc.x; col[(sub * 4 + 1) * T] = acc.y;
    col[(sub * 4 + 2) * T] = acc.z; col[(sub * 4 + 3) * T] = acc.w;
  }
}

// scatter dc (owner's column) into the grid gradient and return d loss / d (ix,iy,iz)
__device__ __forceinline__ void trilerp_coop_bwd(const Grid& g, const Cell& mine, bool active,
                                                 const float* __restrict__ dcol0, int tbase,
                                                 bool need_dx, float gout[3]) {
  const int lane = threadIdx.x & 31, sub = lane & 7, q = lane >> 3;
  gout[0] = gout[1] = gout[2] = 0.f;
#pragma unroll 1
  for (int grp = 0; grp < 8; ++grp) {
    const int owner = grp * 4 + q;
    const int ix = __shfl_sync(0xffffffffu, mine.ix, owner);
    const int iy = __shfl_sync(0xffffffffu, mine.iy, owner);
    const int iz = __shfl_sync(0xffffffffu, mine.iz, owner);
    const float fx = __shfl_sync(0xffffffffu, mine.fx, owner);
    const float fy = __shfl_sync(0xffffffffu, mine.fy, owner);
    const float fz = __shfl_sync(0xffffffffu, mine.fz, owner);
    const int act = __shfl_sync(0xffffffffu, (int)active, owner);
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (act) {
      const float* col = dcol0 + (tbase + owner);
      const float4 d = make_float4(col[(sub * 4 + 0) * T], col[(sub * 4 + 1) * T],
                                   col[(sub * 4 + 2) * T], col[(sub * 4 + 3) * T]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
        const int x = ix + dx, y = iy + dy, z = iz + dz;
        if (x < g.nx && y < g.ny && z < g.nz) {
          const float wx = dx ? fx : 1.f - fx, wy = dy ? fy : 1.f - fy, wz = dz ? fz : 1.f - fz;
          const size_t off = ((size_t)((size_t)z * g.ny + y) * g.nx + x) * 32 + sub * 4;
          if (g.grad) {
            const float w = wx * wy * wz;
            red_add_v4(g.grad + off, w * d.x, w * d.y, w * d.z, w * d.w);
          }
          if (need_dx) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(g.data + off));
            const float s = v.x * d.x + v.y * d.y + v.z * d.z + v.w * d.w;
            gx += (dx ? 1.f : -1.f) * wy * wz * s;
            gy += (dy ? 1.f : -1.f) * wx * wz * s;
            gz += (dz ? 1.f : -1.f) * wx * wy * s;
          }
        }
      }
    }
    if (need_dx) {
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        gx += __shfl_xor_sync(0xffffffffu, gx, o);
        gy += __shfl_xor_sync(0xffffffffu, gy, o);
        gz += __shfl_xor_sync(0xffffffffu, gz, o);
      }
      // owner lanes of this pass are grp*4 + qq; group qq (lanes 8qq..8qq+7) holds their sums
      const float sx = __shfl_sync(0xffffffffu, gx, (lane & 3) * 8);
      const float sy = __shfl_sync(0xffffffffu, gy, (lane & 3) * 8);
      const float sz = __shfl_sync(0xffffffffu, gz, (lane & 3) * 8);
      if ((lane >> 2) == grp) { gout[0] = sx; gout[1] = sy; gout[2] = sz; }
    }
  }
}

// ------------------------------------------------------------ dense ops ---
__device__ __forceinline__ void fma32(float (&acc)[H], float x, const float* __restrict__ wrow) {
  const float4* w = reinterpret_cast<const float4*>(wrow);
#pragma unroll
  for (int j4 = 0; j4 < 8; ++j4) {
    const float4 v = w[j4];
    acc[4 * j4 + 0] = fmaf(x, v.x, acc[4 * j4 + 0]);
    acc[4 * j4 + 1] = fmaf(x, v.y, acc[4 * j4 + 1]);
    acc[4 * j4 + 2] = fmaf(x, v.z, acc[4 * j4 + 2]);
    acc[4 * j4 + 3] = fmaf(x, v.w, acc[4 * j4 + 3]);
  }
}
__device__ __forceinline__ float dot32(const float (&g)[H], const float* __restrict__ wrow) {
  const float4* w = reinterpret_cast<const float4*>(wrow);
  float a0 = 0.f, a1 = 0.f;
#pragma unroll
  for (int j4 = 0; j4 < 8; ++j4) {
    const float4 v = w[j4];
    a0 = fmaf(g[4 * j4 + 0], v.x, a0);
    a1 = fmaf(g[4 * j4 + 1], v.y, a1);
    a0 = fmaf(g[4 * j4 + 2], v.z, a0);
    a1 = fmaf(g[4 * j4 + 3], v.w, a1);
  }
  return a0 + a1;
}
// acc += W^T[0..n) x, x in a shared-memory column (stride T)
static __device__ __noinline__ void dense_col(float (&acc)[H], const float* __restrict__ wT,
                                       const float* __restrict__ col, int n) {
#pragma unroll 2
  for (int i = 0; i < n; ++i) fma32(acc, col[i * T], wT + i * H);
}
// acc += W^T h, h in registers
static __device__ __noinline__ void dense_reg(float (&acc)[H], const float* __restrict__ wT,
                                       const float (&h)[H]) {
#pragma unroll
  for (int i = 0; i < H; ++i) fma32(acc, h[i], wT + i * H);
}
// col[i] += <W^T[i], g>  for i in [0,n)
static __device__ __noinline__ void denseT_col(float* __restrict__ col, const float* __restrict__ wT,
                                        const float (&g)[H], int n) {
#pragma unroll 2
  for (int i = 0; i < n; ++i) col[i * T] += dot32(g, wT + i * H);
}
// out[i] = <W^T[i], g>
static __device__ __noinline__ void denseT_reg(float (&out)[H], const float* __restrict__ wT,
                                        const float (&g)[H]) {
#pragma unroll
  for (int i = 0; i < H; ++i) out[i] = dot32(g, wT + i * H);
}

static __device__ void stage_weights(const XrdNiceDecoder& d, float* sw) {
  const WOff o = woff(d.c_dim);
  const int in[5] = {E, H, H, E + H, H};
  for (int l = 0; l < 5; ++l) {
    for (int q = threadIdx.x; q < in[l] * H; q += blockDim.x) {
      const int i = q / H, j = q % H;
      sw[o.pts[l] + q] = d.pts_w[l][j * in[l] + i];
    }
    for (int q = threadIdx.x; q < d.c_dim * H; q += blockDim.x) {
      const int i = q / H, j = q % H;
      sw[o.fcc[l] + q] = d.fcc_w[l][j * d.c_dim + i];
    }
    for (int q = threadIdx.x; q < H; q += blockDim.x) {
      sw[o.pts_b + l * H + q] = d.pts_b[l][q];
      sw[o.fcc_b + l * H + q] = d.fcc_b[l][q];
    }
  }
  for (int q = threadIdx.x; q < H * 4; q += blockDim.x) {
    const int j = q / 4, k = q % 4;
    sw[o.out + q] = (k < d.n_out) ? d.out_w[k * H + j] : 0.f;
  }
  for (int q = threadIdx.x; q < 3 * E; q += blockDim.x) sw[o.B + q] = d.B[q];
  for (int q = threadIdx.x; q < 4; q += blockDim.x) sw[o.out_b + q] = (q < d.n_out) ? d.out_b[q] : 0.f;
}

// -------------------------------------------------------------- forward ---
static __global__ void __launch_bounds__(T) k_decoder_fwd(const DecParams P) {
  extern __shared__ __align__(16) float smem[];
  const WOff o = woff(P.dec.c_dim);
  float* sw = smem;
  float* ecol = sw + o.total;          // [E][T]
  float* ccol = ecol + E * T;          // [CMAX][T]
  stage_weights(P.dec, sw);
  __syncthreads();
  const int tid = threadIdx.x, tbase = tid & ~31;
  const int n_tiles = (P.P + T - 1) / T;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * T + tid;
    const bool active = p < P.P;
    double pt[3] = {0.0, 0.0, 0.0};
    if (active) point_f64(P, p, pt);
    if (P.ga.data) {
      Cell ca = make_cell(P, P.ga, pt);
      trilerp_coop(P.ga, ca, active, ccol, tbase);
      if (P.gb.data) {
        Cell cb = make_cell(P, P.gb, pt);
        trilerp_coop(P.gb, cb, active, ccol + 32 * T, tbase);
      }
    } else if (active) {
      for (int m = 0; m < P.dec.c_dim; ++m) ccol[m * T + tid] = P.ext_c[(size_t)m * P.P + p];
    }
    __syncwarp();
    if (active) {
    const float sc = P.embed_scale;
    const float pf[3] = {sc * (float)pt[0], sc * (float)pt[1], sc * (float)pt[2]};
    float* e = ecol + tid;
    float* c = ccol + tid;
    const float* Bm = sw + o.B;
#pragma unroll 3
    for (int m = 0; m < E; ++m)
      e[m * T] = sinf(pf[0] * Bm[m] + pf[1] * Bm[E + m] + pf[2] * Bm[2 * E + m]);
    float h[H], acc[H];
    if (P.acts) {
      for (int m = 0; m < E; ++m) P.acts[(size_t)(row_e() + m) * P.Pp + p] = e[m * T];
      for (int m = 0; m < P.dec.c_dim; ++m) P.acts[(size_t)(row_c() + m) * P.Pp + p] = c[m * T];
    }
#pragma unroll 1
    for (int l = 0; l < 5; ++l) {
#pragma unroll
      for (int j = 0; j < H; ++j) acc[j] = sw[o.pts_b + l * H + j];
      if (l == 0 || l == 3) dense_col(acc, sw + o.pts[l], e, E);
      if (l != 0) dense_reg(acc, sw + o.pts[l] + (l == 3 ? E * H : 0), h);
      uint32_t mask = 0;
#pragma unroll
      for (int j = 0; j < H; ++j) {
        mask |= (acc[j] > 0.f) ? (1u << j) : 0u;
        acc[j] = fmaxf(acc[j], 0.f) + sw[o.fcc_b + l * H + j];
      }
      dense_col(acc, sw + o.fcc[l], c, P.dec.c_dim);
#pragma unroll
      for (int j = 0; j < H; ++j) h[j] = acc[j];
      if (P.masks) P.masks[(size_t)l * P.P + p] = mask;
      if (P.acts)
#pragma unroll
        for (int j = 0; j < H; ++j) P.acts[(size_t)(row_h(l) + j) * P.Pp + p] = h[j];
    }
    float ov[4] = {sw[o.out_b], sw[o.out_b + 1], sw[o.out_b + 2], sw[o.out_b + 3]};
#pragma unroll
    for (int j = 0; j < H; ++j) {
      const float4 w = *reinterpret_cast<const float4*>(sw + o.out + j * 4);
      ov[0] = fmaf(h[j], w.x, ov[0]); ov[1] = fmaf(h[j], w.y, ov[1]);
      ov[2] = fmaf(h[j], w.z, ov[2]); ov[3] = fmaf(h[j], w.w, ov[3]);
    }
    for (int k = 0; k < P.dec.n_out; ++k)
      if (P.out[k]) P.out[k][p] = ov[k];
    }
    __syncwarp();  // columns are rewritten by the helper lanes of the next tile
  }
}

// ------------------------------------------------------------- backward ---
static __global__ void __launch_bounds__(T) k_decoder_bwd(const DecParams P) {
  extern __shared__ __align__(16) float smem[];
  const WOff o = woff(P.dec.c_dim);
  float* sw = smem;
  float* ecol = sw + o.total;  // d loss / d embedding
  float* ccol = ecol + E * T;  // d loss / d grid feature
  stage_weights(P.dec, sw);
  __syncthreads();
  const int tid = threadIdx.x, tbase = tid & ~31;
  const int n_tiles = (P.P + T - 1) / T;
  const int cd = P.dec.c_dim;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * T + tid;
    const bool active = p < P.P;
    double pt[3] = {0.0, 0.0, 0.0};
    float* de = ecol + tid;
    float* dc = ccol + tid;
    float dpf[3] = {0.f, 0.f, 0.f};
    if (active) {
      point_f64(P, p, pt);
      for (int m = 0; m < E; ++m) de[m * T] = 0.f;
      for (int m = 0; m < cd; ++m) dc[m * T] = 0.f;
      float dh[H], g[H];
      float dov[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < P.dec.n_out; ++k)
        if (P.dout[k]) dov[k] = P.dout[k][p];
#pragma unroll
      for (int j = 0; j < H; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(sw + o.out + j * 4);
        dh[j] = dov[0] * w.x + dov[1] * w.y + dov[2] * w.z + dov[3] * w.w;
      }
      if (P.acts)
        for (int k = 0; k < 4; ++k) P.acts[(size_t)(row_do(cd) + k) * P.Pp + p] = dov[k];
#pragma unroll 1
      for (int l = 4; l >= 0; --l) {
        if (P.acts)
#pragma unroll
          for (int j = 0; j < H; ++j) P.acts[(size_t)(row_dh(l, cd) + j) * P.Pp + p] = dh[j];
        denseT_col(dc, sw + o.fcc[l], dh, cd);
        const uint32_t mask = P.masks[(size_t)l * P.P + p];
#pragma unroll
        for (int j = 0; j < H; ++j) g[j] = ((mask >> j) & 1u) ? dh[j] : 0.f;
        if (l == 0 || l == 3) denseT_col(de, sw + o.pts[l], g, E);
        if (l != 0) denseT_reg(dh, sw + o.pts[l] + (l == 3 ? E * H : 0), g);
      }
      // embedding backward: e = sin(scale * p B)
      const float sc = P.embed_scale;
      const float pf[3] = {sc * (float)pt[0], sc * (float)pt[1], sc * (float)pt[2]};
      const float* Bm = sw + o.B;
      for (int m = 0; m < E; ++m) {
        const float gm = de[m * T] * cosf(pf[0] * Bm[m] + pf[1] * Bm[E + m] + pf[2] * Bm[2 * E + m]);
        dpf[0] = fmaf(gm, Bm[m], dpf[0]);
        dpf[1] = fmaf(gm, Bm[E + m], dpf[1]);
        dpf[2] = fmaf(gm, Bm[2 * E + m], dpf[2]);
        if (P.acts) P.acts[(size_t)(row_gm(cd) + m) * P.Pp + p] = gm;
      }
#pragma unroll
      for (int d = 0; d < 3; ++d) dpf[d] *= sc;
      if (P.acts)
        for (int d = 0; d < 3; ++d) P.acts[(size_t)(row_pf(cd) + d) * P.Pp + p] = pf[d];
    }
    __syncwarp();
    if (!P.ga.data) {  // Point-SLAM: hand d loss / d feature to the kNN interpolation backward
      if (active) {
        for (int m = 0; m < cd; ++m) P.ext_dc[(size_t)m * P.P + p] = dc[m * T];
        if (P.need_dp)
#pragma unroll
          for (int d = 0; d < 3; ++d) P.dp[(size_t)d * P.P + p] += dpf[d];
      }
      __syncwarp();
      continue;
    }
    Cell ca = make_cell(P, P.ga, pt);
    float gi[3];
    trilerp_coop_bwd(P.ga, ca, active, ccol, tbase, P.need_dp != 0, gi);
    if (active && P.need_dp) {
      // d index / d p = mult * 2 / (bmax - bmin)   (normalize_3d_coordinate, f64 bound)
      const float m3[3] = {ca.mx, ca.my, ca.mz};
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const float gp = (float)((double)(gi[d] * m3[d]) * 2.0 / (P.bmax[d] - P.bmin[d]));
        P.dp[(size_t)d * P.P + p] += gp + dpf[d];
      }
    }
    __syncwarp();
  }
}

cudaError_t launch_decoder(const DecParams& D, bool bwd, cudaStream_t stream) {
  const size_t smem = sizeof(float) * ((size_t)woff(D.dec.c_dim).total + (size_t)(E + CMAX) * T);
  void (*k)(const DecParams) = bwd ? k_decoder_bwd : k_decoder_fwd;
  const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int n_tiles = (D.P + T - 1) / T, sms = num_sms();
  k<<<n_tiles < sms ? n_tiles : sms, T, smem, stream>>>(D);
  return cudaGetLastError();
}

// --------------------------------------------------- coarse level (N6) ---
// MLP_no_xyz (decoder_nice.py:237-320): h = c; 5 x [h = relu(W h + b)], [c, h] re-concatenated
// after block 2, occupancy = w_out h + b_out.  The grid feature c is sampled with the COARSE
// bound (scene bound x model_coarse_bound_enlarge, conv_onet.py:335-337); no positional
// embedding, no fc_c.  The decoder is frozen (pretrained): gradients go to the grid (and rays).
struct CoarseW {
  const float* pts_w[5];  // torch layout [32][in], in = 32, 32, 32, 64, 32
  const float* pts_b[5];
  const float* out_w;     // [1][32]
  const float* out_b;     // [1]
};
constexpr int CW_L3 = 3 * H * H;            // block 3: [64][32]
constexpr int CW_L4 = CW_L3 + 2 * H * H;
constexpr int CW_OUT = CW_L4 + H * H;
constexpr int CW_B = CW_OUT + H;            // biases 5 x 32, then out bias
constexpr int CW_TOTAL = CW_B + 5 * H + 4;

static __device__ void stage_coarse(const CoarseW& w, float* sw) {
  const int in[5] = {H, H, H, 2 * H, H};
  const int off[5] = {0, H * H, 2 * H * H, CW_L3, CW_L4};
  for (int l = 0; l < 5; ++l) {
    for (int q = threadIdx.x; q < in[l] * H; q += blockDim.x) {
      const int i = q / H, j = q % H;
      sw[off[l] + q] = w.pts_w[l][j * in[l] + i];  // transposed: [in][out]
    }
    for (int q = threadIdx.x; q < H; q += blockDim.x) sw[CW_B + l * H + q] = w.pts_b[l][q];
  }
  for (int q = threadIdx.x; q < H; q += blockDim.x) sw[CW_OUT + q] = w.out_w[q];
  if (threadIdx.x == 0) sw[CW_B + 5 * H] = w.out_b[0];
}

template <bool BWD>
static __global__ void __launch_bounds__(T) k_coarse(const DecParams P, const CoarseW W) {
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;
  float* ccol = sw + CW_TOTAL;  // [32][T]: grid feature (fwd) / its gradient (bwd)
  stage_coarse(W, sw);
  __syncthreads();
  const int tid = threadIdx.x, tbase = tid & ~31;
  const int n_tiles = (P.P + T - 1) / T;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * T + tid;
    const bool active = p < P.P;
    double pt[3] = {0.0, 0.0, 0.0};
    if (active) point_f64(P, p, pt);
    const Cell ca = make_cell(P, P.ga, pt);
    float* c = ccol + tid;
    if (!BWD) {
      trilerp_coop(P.ga, ca, active, ccol, tbase);
      __syncwarp();
      if (active) {
        float h[H], acc[H];
#pragma unroll 1
        for (int l = 0; l < 5; ++l) {
#pragma unroll
          for (int j = 0; j < H; ++j) acc[j] = sw[CW_B + l * H + j];
          if (l == 0) dense_col(acc, sw, c, H);
          else if (l == 3) { dense_col(acc, sw + CW_L3, c, H); dense_reg(acc, sw + CW_L3 + H * H, h); }
          else dense_reg(acc, sw + (l == 4 ? CW_L4 : l * H * H), h);
          uint32_t mask = 0;
#pragma unroll
          for (int j = 0; j < H; ++j) {
            mask |= (acc[j] > 0.f) ? (1u << j) : 0u;
            h[j] = fmaxf(acc[j], 0.f);
          }
          if (P.masks) P.masks[(size_t)l * P.P + p] = mask;
        }
        float o = sw[CW_B + 5 * H];
#pragma unroll
        for (int j = 0; j < H; ++j) o = fmaf(h[j], sw[CW_OUT + j], o);
        P.out[0][p] = o;
      }
      __syncwarp();
    } else {
      float dpf[3] = {0.f, 0.f, 0.f};
      if (active) {
        for (int m = 0; m < H; ++m) c[m * T] = 0.f;
        float dh[H], g[H];
        const float dov = P.dout[0][p];
#pragma unroll
        for (int j = 0; j < H; ++j) dh[j] = dov * sw[CW_OUT + j];
#pragma unroll 1
        for (int l = 4; l >= 0; --l) {
          const uint32_t mask = P.masks[(size_t)l * P.P + p];
#pragma unroll
          for (int j = 0; j < H; ++j) g[j] = ((mask >> j) & 1u) ? dh[j] : 0.f;
          if (l == 0) denseT_col(c, sw, g, H);
          else if (l == 3) { denseT_col(c, sw + CW_L3, g, H); denseT_reg(dh, sw + CW_L3 + H * H, g); }
          else denseT_reg(dh, sw + (l == 4 ? CW_L4 : l * H * H), g);
        }
      }
      __syncwarp();
      float gi[3];
      trilerp_coop_bwd(P.ga, ca, active, ccol, tbase, P.need_dp != 0, gi);
      if (active && P.need_dp) {
        const float m3[3] = {ca.mx, ca.my, ca.mz};
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          const float gp = (float)((double)(gi[d] * m3[d]) * 2.0 / (P.bmax[d] - P.bmin[d]));
          P.dp[(size_t)d * P.P + p] += gp + dpf[d];
        }
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------- composite ---
struct CompParams {
  int R, S;
  const double* z;
  const float *rays_o, *rays_d, *target_s, *target_d;
  double bmin[3], bmax[3];
  const float *occ_a, *occ_b;  // occupancy logit = occ_a + (occ_b ? occ_b : 0)
  const float* rgb[3];         // may be NULL (stages middle / fine)
  // outputs
  float* o_rgb; double* o_depth; double* o_var; float* o_raw;
  // backward
  const float* gd;   // [R]   d loss / d depth
  const float* gc;   // [R][3]
  float* d_occ;      // [P]
  float* d_rgb[3];   // [P]
  float* o_w;        // [R][S] k_composite<false, .., true>: the weights alone
};

__device__ __forceinline__ bool in_bound(const CompParams& P, int r, double z) {
  bool ok = true;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double pt = __dadd_rn((double)P.rays_o[r * 3 + d], __dmul_rn((double)P.rays_d[r * 3 + d], z));
    ok = ok && (pt < P.bmax[d]) && (pt > P.bmin[d]);
  }
  return ok;
}

// warp per ray, S <= 32 NS: lane handles samples lane + 32 s, s < NS (NS = 2: S <= 64, NS = 4:
// S <= 128).  WEIGHTS (forward only): pass 1 of importance sampling, which needs the weights
// [R][S] alone and writes nothing else.
template <bool BWD, int NS, bool WEIGHTS>
static __global__ void __launch_bounds__(128) k_composite(const CompParams P) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + warp;
  if (r >= P.R) return;
  const int S = P.S;
  float alpha[NS], col[NS][3], w[NS], Tt[NS];
  double z[NS];
  bool inb[NS], have[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const int k = lane + 32 * s;
    have[s] = k < S;
    alpha[s] = 0.f; z[s] = 0.0; inb[s] = false;
    col[s][0] = col[s][1] = col[s][2] = 0.f;
    if (have[s]) {
      const size_t p = (size_t)r * S + k;
      z[s] = P.z[p];
      inb[s] = in_bound(P, r, z[s]);
      float occ = P.occ_a[p] + (P.occ_b ? P.occ_b[p] : 0.f);
      if (!inb[s]) occ = 100.f;  // eval_points: ret[~mask, 3] = 100
      alpha[s] = sigmoidf_acc(10.f * occ);
#pragma unroll
      for (int c = 0; c < 3; ++c) col[s][c] = P.rgb[c] ? P.rgb[c][p] : 0.f;
      if (!BWD && !WEIGHTS && P.o_raw) {
        float4 rw = make_float4(col[s][0], col[s][1], col[s][2], occ);
        *reinterpret_cast<float4*>(P.o_raw + p * 4) = rw;
      }
    }
  }
  // exclusive product of (1 - alpha + 1e-10) in sample order (torch.cumprod, f32)
  float run = 1.f;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const float f = have[s] ? (1.f - alpha[s] + 1e-10f) : 1.f;
    float inc = f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc *= v;
    }
    float exc = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) exc = 1.f;
    Tt[s] = run * exc;
    run *= __shfl_sync(0xffffffffu, inc, 31);
    w[s] = alpha[s] * Tt[s];
  }
  if (WEIGHTS) {
#pragma unroll
    for (int s = 0; s < NS; ++s)
      if (have[s]) P.o_w[(size_t)r * S + lane + 32 * s] = w[s];
    return;
  }
  double depth = 0.0;
  float cr[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int s = 0; s < NS; ++s)
    if (have[s]) {
      depth += (double)w[s] * z[s];
#pragma unroll
      for (int c = 0; c < 3; ++c) cr[c] = fmaf(w[s], col[s][c], cr[c]);
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    depth += __shfl_xor_sync(0xffffffffu, depth, o);
#pragma unroll
    for (int c = 0; c < 3; ++c) cr[c] += __shfl_xor_sync(0xffffffffu, cr[c], o);
  }
  if (!BWD) {
    double var = 0.0;
#pragma unroll
    for (int s = 0; s < NS; ++s)
      if (have[s]) { const double t = z[s] - depth; var += (double)w[s] * t * t; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    if (lane == 0) {
      P.o_depth[r] = depth; P.o_var[r] = var;
      P.o_rgb[r * 3] = cr[0]; P.o_rgb[r * 3 + 1] = cr[1]; P.o_rgb[r * 3 + 2] = cr[2];
    }
    return;
  }
  // backward: q_k = gd z_k + <gc, c_k>;  dL/dalpha_k = q_k T_k - (sum_{j>k} q_j w_j)/(1-alpha_k+eps)
  const float gd = P.gd[r];
  const float gcx = P.gc[r * 3], gcy = P.gc[r * 3 + 1], gcz = P.gc[r * 3 + 2];
  float qw[NS], q[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    q[s] = have[s] ? (float)((double)gd * z[s]) + gcx * col[s][0] + gcy * col[s][1] + gcz * col[s][2] : 0.f;
    qw[s] = q[s] * w[s];
  }
  // suffix sums (exclusive) over the 32 NS slots: above[s] = the totals of the slots above s
  float above[NS];
  above[NS - 1] = 0.f;
#pragma unroll
  for (int s = NS - 2; s >= 0; --s) {
    float tot = qw[s + 1];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    above[s] = s == NS - 2 ? tot : tot + above[s + 1];
  }
  float suf[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    float inc = qw[s];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_down_sync(0xffffffffu, inc, o);
      if (lane + o < 32) inc += v;
    }
    float exc = __shfl_down_sync(0xffffffffu, inc, 1);
    if (lane == 31) exc = 0.f;
    suf[s] = exc + above[s];
  }
#pragma unroll
  for (int s = 0; s < NS; ++s)
    if (have[s]) {
      const size_t p = (size_t)r * S + lane + 32 * s;
      const float da = q[s] * Tt[s] - suf[s] / (1.f - alpha[s] + 1e-10f);
      P.d_occ[p] = inb[s] ? da * 10.f * alpha[s] * (1.f - alpha[s]) : 0.f;
      if (P.d_rgb[0]) {
        P.d_rgb[0][p] = gcx * w[s]; P.d_rgb[1][p] = gcy * w[s]; P.d_rgb[2][p] = gcz * w[s];
      }
    }
}

// the instantiation for S samples per ray (two or four slots per lane)
template <bool BWD>
static cudaError_t launch_composite(const CompParams& C, cudaStream_t stream) {
  if (C.S <= 64) k_composite<BWD, 2, false><<<(C.R + 3) / 4, 128, 0, stream>>>(C);
  else k_composite<BWD, 4, false><<<(C.R + 3) / 4, 128, 0, stream>>>(C);
  return cudaGetLastError();
}

// ------------------------------------------------------------- sample_pdf ---
// Importance samples of pass 2 (conv_onet.py:498-506), one warp per ray: sample_pdf
// (sample_pdf.cuh, shared with Co-SLAM's k_importance) with float64 bins and samples on pass 1's
// composite weights (k_composite<.., WEIGHTS>), z_out = sort(z ++ samples).
struct PdfParams {
  int R, S, N;        // S: pass 1's samples per ray, N: importance samples per ray
  const float* w;     // [R][S] pass 1's weights
  const double* z;    // [R][S] pass 1's sorted samples
  const float* u;     // [R][N] uniforms, or NULL
  const float* lin_u; // [N] the det linspace (u NULL, det)
  int det;
  uint64_t seed;      // u NULL, !det: Philox at counters 2^63 + r N + j
  double* z_out;      // [R][S + N]
  double* z_samples;  // [R][N] the samples in draw order, or NULL
};
constexpr int kPdfS = 64, kPdfT = 128;  // limits of pass 1 and of the merge

static __global__ void __launch_bounds__(128) k_sample_pdf(const PdfParams p) {
  __shared__ float s_pdf[4][kPdfS], s_cdf[4][kPdfS];
  __shared__ double s_bins[4][kPdfS], s_z[4][kPdfT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + warp;
  if (r >= p.R) return;  // warp-uniform
  const int S = p.S, N = p.N;
  const float* wr = p.w + (size_t)r * S;
  pdf_cdf([&](int j) { return wr[j]; }, p.z + (size_t)r * S, S, s_pdf[warp], s_cdf[warp],
          s_bins[warp], s_z[warp], lane);
  invert_cdf(PdfDraw{p.u, p.lin_u, p.det, p.seed}, r, S, N, s_cdf[warp], s_bins[warp], s_z[warp],
             p.z_samples ? p.z_samples + (size_t)r * N : nullptr, lane);
  rank_merge(s_z[warp], S + N, p.z_out + (size_t)r * (S + N), lane);
}

// ------------------------------------------------------------------ loss ---
struct LossParams {
  int R, is_mapping, with_color, handle_dynamic, use_color_in_tracking;
  float w_color;
  const float *target_s, *target_d, *rgb;
  const double *depth, *var;
  float* gd; float* gc;   // per-ray coefficients
  double* tmp;            // [R] scratch (tracking)
  float* losses;          // [2]
};

static __global__ void __launch_bounds__(1024) k_loss(const LossParams P) {
  __shared__ double red[2][32];
  __shared__ double s_med;
  const int tid = threadIdx.x;
  double ld = 0.0, lc = 0.0;
  if (P.is_mapping) {
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float D = P.target_d[r];
      const double d = P.depth[r];
      float gd = 0.f;
      if (D > 0.f) { ld += fabs((double)D - d); gd = (d > (double)D) ? 1.f : ((d < (double)D) ? -1.f : 0.f); }
      P.gd[r] = gd;
      for (int c = 0; c < 3; ++c) {
        float g = 0.f;
        if (P.with_color) {
          const float df = P.target_s[r * 3 + c] - P.rgb[r * 3 + c];
          lc += (double)fabsf(df);
          g = (df < 0.f) ? P.w_color : ((df > 0.f) ? -P.w_color : 0.f);
        }
        P.gc[r * 3 + c] = g;
      }
    }
    lc *= (double)P.w_color;
  } else {
    // tmp = |D - depth| / sqrt(var + 1e-10); mask = tmp < 10 median(tmp) & D > 0
    for (int r = tid; r < P.R; r += blockDim.x)
      P.tmp[r] = fabs((double)P.target_d[r] - P.depth[r]) / sqrt(P.var[r] + 1e-10);
    __syncthreads();
    if (P.handle_dynamic) {
      const int want = (P.R - 1) / 2;  // torch.median: lower median
      for (int r = tid; r < P.R; r += blockDim.x) {
        const double v = P.tmp[r];
        int rank = 0;
        for (int j = 0; j < P.R; ++j) {
          const double u = P.tmp[j];
          rank += (u < v) || (u == v && j < r);
        }
        if (rank == want) s_med = v;
      }
    }
    __syncthreads();
    for (int r = tid; r < P.R; r += blockDim.x) {
      const float D = P.target_d[r];
      const double t = P.tmp[r], d = P.depth[r];
      const bool m = (P.handle_dynamic ? (t < 10.0 * s_med) : true) && (D > 0.f);
      float gd = 0.f;
      if (m) {
        ld += t;
        const double inv = 1.0 / sqrt(P.var[r] + 1e-10);
        gd = (float)((d > (double)D) ? inv : ((d < (double)D) ? -inv : 0.0));
      }
      P.gd[r] = gd;
      for (int c = 0; c < 3; ++c) {
        float g = 0.f;
        if (m && P.use_color_in_tracking) {
          const float df = P.target_s[r * 3 + c] - P.rgb[r * 3 + c];
          lc += (double)fabsf(df);
          g = (df < 0.f) ? P.w_color : ((df > 0.f) ? -P.w_color : 0.f);
        }
        P.gc[r * 3 + c] = g;
      }
    }
    lc *= (double)P.w_color;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ld += __shfl_xor_sync(0xffffffffu, ld, o);
    lc += __shfl_xor_sync(0xffffffffu, lc, o);
  }
  if ((tid & 31) == 0) { red[0][tid >> 5] = ld; red[1][tid >> 5] = lc; }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[0][i]; b += red[1][i]; }
    P.losses[0] = (float)a;
    P.losses[1] = (float)b;
  }
}

// --------------------------------------------------------- ray reduction ---
static __global__ void __launch_bounds__(128) k_rayreduce(int R, int S, int P, const double* z,
                                                   const float* dp, float* d_o, float* d_d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + warp;
  if (r >= R) return;
  float a[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = lane; k < S; k += 32) {
    const size_t p = (size_t)r * S + k;
    const double zz = z[p];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float g = dp[(size_t)d * P + p];
      a[d] += g;
      a[3 + d] += (float)((double)g * zz);
    }
  }
#pragma unroll
  for (int d = 0; d < 6; ++d) a[d] = warp_sum(a[d]);
  if (lane == 0)
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      if (d_o) d_o[r * 3 + d] = a[d];
      if (d_d) d_d[r * 3 + d] = a[3 + d];
    }
}

}  // namespace nice
}  // namespace xrd

using namespace xrd;
using namespace xrd::nice;

namespace {
struct Ws : Carver {
  Ws(void* base, int R, int S, int with_grads)
      : Carver(base), R(R), P((size_t)R * S), g(with_grads != 0) {}
  const size_t R, P;
  const bool g;
  float* maxd = take<float>(1);  // alone in a 256-byte header
  double* z = take<double>(P);
  float *occ_mid = take<float>(P), *occ_fine = take<float>(P), *rgb = take<float>(3 * P);
  double *depth = take<double>(R), *var = take<double>(R);  // per-ray rows, reserved and unused
  float* orgb = take<float>(R * 3);
  // with_grads only
  float *d_occ = g ? take<float>(P) : nullptr, *d_rgb = g ? take<float>(3 * P) : nullptr;
  uint32_t* masks = g ? take<uint32_t>(3 * 5 * P) : nullptr;
  float* dp = g ? take<float>(3 * P) : nullptr;
  float *gd = g ? take<float>(R) : nullptr, *gc = g ? take<float>(R * 3) : nullptr;
  double* tmp = g ? take<double>(R) : nullptr;
  float* acts = g ? take<float>((size_t)n_rows(32) * align_up(P, 64)) : nullptr;
  // importance sampling, pass 1 (S0 < S samples per ray): its sorted samples z1 [R*S0] f64
  // and weights w1 [R*S0] f32 live in the rgb rows [3P] f32, which pass 1 does not decode into
  // and pass 2 writes only after k_sample_pdf has read them (2 R S0 + R S0 floats <= 3P)
  double* z1 = reinterpret_cast<double*>(rgb);
  float* w1 = rgb + 2 * P;
};

// rendering_perturb / rendering_n_importance of one call (the trailing fields of XrdNiceCfg and
// XrdNiceCoarseCfg); -> XRD_OK or the status to return
struct Sampling {
  int S0, N, S;  // pass 1, importance, total samples per ray
  bool perturb;
  int check() const {
    if (N < 0 || S0 > kPdfS || S > kPdfT) return XRD_E_SHAPE;
    return XRD_OK;
  }
};

template <class Cfg>
static Sampling sampling(const Cfg* cfg, int S0) {
  Sampling m;
  m.S0 = S0; m.N = cfg->n_importance; m.S = S0 + (m.N > 0 ? m.N : 0);
  m.perturb = cfg->perturb > 0.f;
  return m;
}

static cudaError_t launch_sample(const SampleParams& sp, bool perturb, cudaStream_t stream) {
  if (perturb) k_sample<true><<<(sp.R + 3) / 4, 128, 0, stream>>>(sp);
  else k_sample<false><<<(sp.R + 3) / 4, 128, 0, stream>>>(sp);
  return cudaGetLastError();
}

// pass 1's weights (k_composite over the S0 samples at z1, occupancies already decoded) and
// sample_pdf -> the merged samples z [R][S0 + N]
template <class Cfg>
static cudaError_t importance(CompParams C, const Cfg* cfg, const Sampling& m, const Ws& L,
                              double* z, cudaStream_t stream) {
  C.z = L.z1; C.S = m.S0; C.o_w = L.w1;
  k_composite<false, 2, true><<<(C.R + 3) / 4, 128, 0, stream>>>(C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  PdfParams q;
  q.R = C.R; q.S = m.S0; q.N = m.N; q.w = L.w1; q.z = L.z1;
  q.u = cfg->importance_u; q.lin_u = cfg->t_importance; q.det = cfg->perturb == 0.f;
  q.seed = cfg->seed; q.z_out = z; q.z_samples = nullptr;
  k_sample_pdf<<<(C.R + 3) / 4, 128, 0, stream>>>(q);
  return cudaGetLastError();
}
}  // namespace

extern "C" size_t xrd_nice_workspace_bytes(int n_rays, int n_samples_total, int with_grads) {
  return Ws(nullptr, n_rays, n_samples_total, with_grads).bytes();
}

extern "C" int xrd_nice_step(const XrdRays* rays, const XrdNiceGrid grids[3],
                             const XrdNiceDecoder decoders[3], const XrdNiceCfg* cfg,
                             XrdNiceOut* out, XrdNiceGrads* grads, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  if (!rays || !grids || !decoders || !cfg || !out || !workspace) return XRD_E_NULL;
  if (!rays->rays_o || !rays->rays_d || !rays->target_d) return XRD_E_NULL;
  if (!out->rgb || !out->depth || !out->uncertainty) return XRD_E_NULL;
  const Sampling m = sampling(cfg, cfg->n_samples + cfg->n_surface);
  const int R = rays->n_rays, S = m.S;
  if (R <= 0) return XRD_OK;
  if (m.S0 < 2 || m.S0 > 64 || cfg->n_samples < 2 || cfg->n_surface < 2) return XRD_E_SHAPE;
  if (int st = m.check()) return st;
  if (m.N > 0 && !cfg->importance_u && !m.perturb && !cfg->t_importance) return XRD_E_NULL;
  if (cfg->stage < XRD_NICE_MIDDLE || cfg->stage > XRD_NICE_COLOR) return XRD_E_SHAPE;
  if (!cfg->t_uniform || !cfg->t_surface) return XRD_E_NULL;
  if (decoders[0].c_dim != 32 || decoders[1].c_dim != 64 || decoders[2].c_dim != 32) return XRD_E_SHAPE;
  if (decoders[0].n_out != 1 || decoders[1].n_out != 1 || decoders[2].n_out != 4) return XRD_E_SHAPE;
  if (grads && (!rays->target_s || !out->losses)) return XRD_E_NULL;
  if (grads && !cfg->is_mapping && R > 8192) return XRD_E_SHAPE;  // single-block median
  const Ws L(workspace, R, S, grads != nullptr);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = R * S, Pp = (int)align_up((size_t)P, 64);
  double* z = out->z_vals ? out->z_vals : L.z;
  float* occ_mid = L.occ_mid;
  float* occ_fine = L.occ_fine;
  float* rgb = L.rgb;
  const int stage = cfg->stage;

  if (!cfg->max_depth_global) {
    k_maxdepth<<<1, 1024, 0, stream>>>(rays->target_d, R, L.maxd);
    XRD_LAUNCH_CHECK();
  }
  SampleParams sp;
  sp.R = R; sp.ns = cfg->n_samples; sp.nsurf = cfg->n_surface; sp.no_depth = 0;
  sp.rays_o = rays->rays_o; sp.rays_d = rays->rays_d; sp.target_d = rays->target_d;
  for (int d = 0; d < 3; ++d) { sp.bmin[d] = cfg->bound_min[d]; sp.bmax[d] = cfg->bound_max[d]; }
  sp.maxd = cfg->max_depth_global ? cfg->max_depth_global : L.maxd; sp.z = z;
  sp.t_uniform = cfg->t_uniform; sp.t_surface = cfg->t_surface;
  sp.noise = cfg->perturb_u; sp.seed = cfg->seed;
  if (m.N > 0) sp.z = L.z1;
  XRD_CUDA_TRY(launch_sample(sp, m.perturb, stream));

  const bool train_color = grads && grads->d_color && stage == XRD_NICE_COLOR;
  auto dec_params = [&](int d) {
    DecParams D;
    D.P = P; D.S = S; D.z = z; D.rays_o = rays->rays_o; D.rays_d = rays->rays_d;
    for (int k = 0; k < 3; ++k) { D.bmin[k] = cfg->bound_min[k]; D.bmax[k] = cfg->bound_max[k]; }
    D.ga = {grids[d].data, grads ? grads->d_grid[d] : nullptr, grids[d].nx, grids[d].ny, grids[d].nz};
    if (d == 1) D.gb = {grids[0].data, nullptr, grids[0].nx, grids[0].ny, grids[0].nz};
    D.dec = decoders[d];
    D.masks = grads ? L.masks + (size_t)d * 5 * P : nullptr;
    if (d == 2 && train_color) { D.acts = L.acts; D.Pp = Pp; }
    D.dp = L.dp;
    D.need_dp = grads && (grads->d_rays_o || grads->d_rays_d);
    return D;
  };

  CompParams C;
  C.R = R; C.S = S; C.z = z; C.rays_o = rays->rays_o; C.rays_d = rays->rays_d;
  C.target_s = rays->target_s; C.target_d = rays->target_d;
  for (int d = 0; d < 3; ++d) { C.bmin[d] = cfg->bound_min[d]; C.bmax[d] = cfg->bound_max[d]; }
  C.occ_a = occ_mid; C.occ_b = stage >= XRD_NICE_FINE ? occ_fine : nullptr;
  for (int c = 0; c < 3; ++c) C.rgb[c] = stage == XRD_NICE_COLOR ? rgb + (size_t)c * P : nullptr;
  C.o_rgb = out->rgb; C.o_depth = out->depth; C.o_var = out->uncertainty; C.o_raw = out->raw;
  C.gd = nullptr; C.gc = nullptr; C.d_occ = nullptr; C.d_rgb[0] = C.d_rgb[1] = C.d_rgb[2] = nullptr;
  C.o_w = nullptr;

  if (m.N > 0) {
    // pass 1 (conv_onet.py:483-496): decoders and weights over the S0 samples at z1, no loss,
    // no backward; its outputs are dropped
    const int P1 = R * m.S0;
    for (int d = 0; d <= (stage < XRD_NICE_FINE ? stage : XRD_NICE_FINE); ++d) {
      DecParams D = dec_params(d);
      D.P = P1; D.S = m.S0; D.z = L.z1; D.masks = nullptr; D.acts = nullptr; D.need_dp = 0;
      if (d == 0) D.out[0] = occ_mid;
      if (d == 1) D.out[0] = occ_fine;
      XRD_CUDA_TRY(launch_decoder(D, false, stream));
    }
    CompParams C1 = C;
    for (int c = 0; c < 3; ++c) C1.rgb[c] = nullptr;  // the weights need occupancies only: no
                                                      // colour decoder in pass 1
    XRD_CUDA_TRY(importance(C1, cfg, m, L, z, stream));
  }

  for (int d = 0; d <= stage; ++d) {
    DecParams D = dec_params(d);
    if (d == 0) D.out[0] = occ_mid;
    if (d == 1) D.out[0] = occ_fine;
    if (d == 2) { D.out[0] = rgb; D.out[1] = rgb + P; D.out[2] = rgb + 2 * (size_t)P; }
    KernelTimer kt(stream);
    XRD_CUDA_TRY(launch_decoder(D, false, stream));
  }

  XRD_CUDA_TRY(launch_composite<false>(C, stream));
  if (!grads) return XRD_OK;

  LossParams LP;
  LP.R = R; LP.is_mapping = cfg->is_mapping; LP.with_color = stage == XRD_NICE_COLOR;
  LP.handle_dynamic = cfg->handle_dynamic; LP.use_color_in_tracking = cfg->use_color_in_tracking;
  LP.w_color = cfg->w_color; LP.target_s = rays->target_s; LP.target_d = rays->target_d;
  LP.rgb = out->rgb; LP.depth = out->depth; LP.var = out->uncertainty;
  LP.gd = L.gd; LP.gc = L.gc;
  LP.tmp = L.tmp; LP.losses = out->losses;
  k_loss<<<1, 1024, 0, stream>>>(LP);
  XRD_LAUNCH_CHECK();

  C.gd = LP.gd; C.gc = LP.gc;
  C.d_occ = L.d_occ;
  if (stage == XRD_NICE_COLOR)
    for (int c = 0; c < 3; ++c) C.d_rgb[c] = L.d_rgb + (size_t)c * P;
  XRD_CUDA_TRY(launch_composite<true>(C, stream));

  XRD_CUDA_TRY(cudaMemsetAsync(L.dp, 0, 3 * (size_t)P * 4, stream));
  for (int d = 0; d <= stage; ++d) {
    DecParams D = dec_params(d);
    if (d < 2) D.dout[0] = C.d_occ;
    else { D.dout[0] = C.d_rgb[0]; D.dout[1] = C.d_rgb[1]; D.dout[2] = C.d_rgb[2]; }
    XRD_CUDA_TRY(launch_decoder(D, true, stream));
  }

  if (train_color) {
    const XrdNiceDecoderGrads* G = grads->d_color;
    const float* A = L.acts;
    const uint32_t* mk = L.masks + (size_t)2 * 5 * P;
    const int cd = 32;
    DwParams Q;
    Q.n_jobs = 0; Q.P = P; Q.Pp = Pp;
    Q.chunk = 512;
    auto rowp = [&](int row) { return A + (size_t)row * Pp; };
    auto add = [&](const float* a, int nA, const float* b, int nB, const uint32_t* m, float* o,
                   int sj, int si, float* bias) {
      if (!o) return;
      DwJob& J = Q.jobs[Q.n_jobs++];
      J.A = a; J.nA = nA; J.B = b; J.nB = nB; J.mask = m; J.out = o; J.sj = sj; J.si = si; J.bias = bias;
    };
    const int in[5] = {E, H, H, E + H, H};
    for (int l = 0; l < 5; ++l) {
      const float* dh = rowp(row_dh(l, cd));
      const uint32_t* m = mk + (size_t)l * P;
      if (l == 0) add(rowp(row_e()), E, dh, H, m, G->pts_w[0], in[0], 1, G->pts_b[0]);
      else if (l == 3) {
        add(rowp(row_e()), E, dh, H, m, G->pts_w[3], in[3], 1, G->pts_b[3]);
        add(rowp(row_h(2)), H, dh, H, m, G->pts_w[3] ? G->pts_w[3] + E : nullptr, in[3], 1, nullptr);
      } else add(rowp(row_h(l - 1)), H, dh, H, m, G->pts_w[l], in[l], 1, G->pts_b[l]);
      add(rowp(row_c()), cd, dh, H, nullptr, G->fcc_w[l], cd, 1, G->fcc_b[l]);
    }
    add(rowp(row_h(4)), H, rowp(row_do(cd)), 4, nullptr, G->out_w, H, 1, G->out_b);
    // embedder: dB[k][m] = sum_p pf[k] gm[m]  (A = gm rows, B = pf rows)
    add(rowp(row_gm(cd)), E, rowp(row_pf(cd)), 3, nullptr, G->B, E, 1, nullptr);
    if (Q.n_jobs > DW_MAX_JOBS) return XRD_E_SHAPE;
    XRD_CUDA_TRY(launch_dw(Q, stream));
  }
  if (grads->d_rays_o || grads->d_rays_d) {
    k_rayreduce<<<(R + 3) / 4, 128, 0, stream>>>(R, S, P, z, L.dp, grads->d_rays_o,
                                                 grads->d_rays_d);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}

extern "C" int xrd_nice_sample_pdf(int n_rays, int n_samples, int n_importance,
                                   const float* weights, const double* z_vals, const float* u,
                                   const float* t_importance, int det, uint64_t seed,
                                   double* z_out, double* z_samples, void* stream_) {
  if (!weights || !z_vals || !z_out) return XRD_E_NULL;
  if (n_rays <= 0 || n_importance <= 0) return XRD_OK;
  if (n_samples < 2 || n_samples > kPdfS || n_samples + n_importance > kPdfT) return XRD_E_SHAPE;
  if (!u && det && !t_importance) return XRD_E_NULL;
  PdfParams q;
  q.R = n_rays; q.S = n_samples; q.N = n_importance; q.w = weights; q.z = z_vals;
  q.u = u; q.lin_u = t_importance; q.det = det; q.seed = seed; q.z_out = z_out;
  q.z_samples = z_samples;
  k_sample_pdf<<<(n_rays + 3) / 4, 128, 0, (cudaStream_t)stream_>>>(q);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

// ---- mesher queries (conv_onet.py:213-240 query_fn / color_func): NICE.forward at free points
static __global__ void k_query_pack(int P, const float* occ_mid, const float* occ_fine,
                                    const float* rgb, float* raw) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float4 o = make_float4(0.f, 0.f, 0.f, occ_mid[p] + (occ_fine ? occ_fine[p] : 0.f));
  if (rgb) { o.x = rgb[p]; o.y = rgb[P + p]; o.z = rgb[2 * (size_t)P + p]; }
  *reinterpret_cast<float4*>(raw + (size_t)p * 4) = o;
}

struct QueryWs : Carver {
  QueryWs(void* base, int n_points) : Carver(base), P((size_t)n_points) {}
  const size_t P;
  double* z = take<double>(P);
  float *zero_d = take<float>(3 * P), *occ_mid = take<float>(P), *occ_fine = take<float>(P);
  float* rgb = take<float>(3 * P);
};

extern "C" size_t xrd_nice_query_workspace_bytes(int n_points) {
  return QueryWs(nullptr, n_points).bytes();
}

extern "C" int xrd_nice_query(const float* points, int n_points, const XrdNiceGrid grids[3],
                              const XrdNiceDecoder decoders[3], const double bound_min[3],
                              const double bound_max[3], int stage, float* raw, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  if (!points || !grids || !decoders || !bound_min || !bound_max || !raw || !workspace) return XRD_E_NULL;
  if (n_points <= 0) return XRD_OK;
  if (stage < XRD_NICE_MIDDLE || stage > XRD_NICE_COLOR) return XRD_E_SHAPE;
  const QueryWs L(workspace, n_points);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = n_points;
  // point = rays_o + rays_d * z with rays_o = the query point, rays_d = 0, z = 0 (exact)
  XRD_CUDA_TRY(cudaMemsetAsync(L.z, 0, (size_t)P * 8, stream));
  XRD_CUDA_TRY(cudaMemsetAsync(L.zero_d, 0, (size_t)P * 12, stream));
  for (int d = 0; d <= stage; ++d) {
    DecParams D;
    D.P = P; D.S = 1; D.z = L.z; D.rays_o = points; D.rays_d = L.zero_d;
    for (int k = 0; k < 3; ++k) { D.bmin[k] = bound_min[k]; D.bmax[k] = bound_max[k]; }
    D.ga = {grids[d].data, nullptr, grids[d].nx, grids[d].ny, grids[d].nz};
    if (d == 1) D.gb = {grids[0].data, nullptr, grids[0].nx, grids[0].ny, grids[0].nz};
    D.dec = decoders[d];
    if (d == 0) D.out[0] = L.occ_mid;
    if (d == 1) D.out[0] = L.occ_fine;
    if (d == 2) { D.out[0] = L.rgb; D.out[1] = L.rgb + P; D.out[2] = L.rgb + 2 * (size_t)P; }
    XRD_CUDA_TRY(launch_decoder(D, false, stream));
  }
  k_query_pack<<<(P + 255) / 256, 256, 0, stream>>>(P, L.occ_mid,
                                                    stage >= XRD_NICE_FINE ? L.occ_fine : nullptr,
                                                    stage == XRD_NICE_COLOR ? L.rgb : nullptr, raw);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" size_t xrd_nice_coarse_workspace_bytes(int n_rays, int n_samples, int with_grads) {
  return Ws(nullptr, n_rays, n_samples, with_grads).bytes();
}

// Stage 'coarse' (conv_onet.py:137-138,397-402; decoder_nice.py:389-393): 32 uniform samples up
// to the bound exit, MLP_no_xyz on the coarse grid, occupancy compositing, mapping depth loss,
// gradient w.r.t. the coarse grid (and the rays).
extern "C" int xrd_nice_coarse_step(const XrdRays* rays, const XrdNiceGrid* grid,
                                    const XrdNiceCoarseDecoder* dec, const XrdNiceCoarseCfg* cfg,
                                    XrdNiceOut* out, float* d_grid, float* d_rays_o, float* d_rays_d,
                                    int with_grads, void* workspace, size_t workspace_bytes,
                                    void* stream_) {
  if (!rays || !grid || !dec || !cfg || !out || !workspace) return XRD_E_NULL;
  if (!rays->rays_o || !rays->rays_d || !grid->data || !cfg->t_uniform) return XRD_E_NULL;
  if (!out->rgb || !out->depth || !out->uncertainty) return XRD_E_NULL;
  if (with_grads && (!rays->target_d || !out->losses)) return XRD_E_NULL;
  const Sampling m = sampling(cfg, cfg->n_samples);
  const int R = rays->n_rays, S = m.S;
  if (R <= 0) return XRD_OK;
  if (m.S0 < 2 || m.S0 > 64) return XRD_E_SHAPE;
  if (int st = m.check()) return st;
  if (m.N > 0 && !cfg->importance_u && !m.perturb && !cfg->t_importance) return XRD_E_NULL;
  const Ws L(workspace, R, S, with_grads);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = R * S;
  double* z = out->z_vals ? out->z_vals : L.z;
  float* occ = L.occ_mid;

  SampleParams sp;
  sp.R = R; sp.ns = m.S0; sp.nsurf = 0; sp.no_depth = 1;
  sp.rays_o = rays->rays_o; sp.rays_d = rays->rays_d; sp.target_d = nullptr;
  for (int d = 0; d < 3; ++d) { sp.bmin[d] = cfg->bound_min[d]; sp.bmax[d] = cfg->bound_max[d]; }
  sp.maxd = nullptr; sp.z = m.N > 0 ? L.z1 : z; sp.t_uniform = cfg->t_uniform; sp.t_surface = nullptr;
  sp.noise = cfg->perturb_u; sp.seed = cfg->seed;
  XRD_CUDA_TRY(launch_sample(sp, m.perturb, stream));

  DecParams D;
  D.P = P; D.S = S; D.z = z; D.rays_o = rays->rays_o; D.rays_d = rays->rays_d;
  for (int k = 0; k < 3; ++k) { D.bmin[k] = cfg->coarse_bound_min[k]; D.bmax[k] = cfg->coarse_bound_max[k]; }
  D.ga = {grid->data, with_grads ? d_grid : nullptr, grid->nx, grid->ny, grid->nz};
  D.out[0] = occ;
  D.masks = L.masks;
  D.dp = L.dp;
  D.need_dp = with_grads && (d_rays_o || d_rays_d);
  CoarseW W;
  for (int l = 0; l < 5; ++l) { W.pts_w[l] = dec->pts_w[l]; W.pts_b[l] = dec->pts_b[l]; }
  W.out_w = dec->out_w; W.out_b = dec->out_b;
  const size_t smem = sizeof(float) * ((size_t)CW_TOTAL + (size_t)H * T);
  const int n_tiles = (P + T - 1) / T;
  const int sms = num_sms();
  const int gridx = n_tiles < sms ? n_tiles : sms;
  XRD_CUDA_TRY(cudaFuncSetAttribute(k_coarse<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CompParams C;
  C.R = R; C.S = S; C.z = z; C.rays_o = rays->rays_o; C.rays_d = rays->rays_d;
  C.target_s = rays->target_s; C.target_d = rays->target_d;
  for (int d = 0; d < 3; ++d) { C.bmin[d] = cfg->bound_min[d]; C.bmax[d] = cfg->bound_max[d]; }
  C.occ_a = occ; C.occ_b = nullptr;
  for (int c = 0; c < 3; ++c) C.rgb[c] = nullptr;
  C.o_rgb = out->rgb; C.o_depth = out->depth; C.o_var = out->uncertainty; C.o_raw = out->raw;
  C.gd = nullptr; C.gc = nullptr; C.d_occ = nullptr; C.d_rgb[0] = C.d_rgb[1] = C.d_rgb[2] = nullptr;
  C.o_w = nullptr;
  if (m.N > 0) {  // pass 1 over the S0 samples at z1, forward only
    DecParams D1 = D;
    D1.P = R * m.S0; D1.S = m.S0; D1.z = L.z1; D1.masks = nullptr; D1.need_dp = 0;
    D1.ga.grad = nullptr;
    const int t1 = (D1.P + T - 1) / T;
    k_coarse<false><<<t1 < sms ? t1 : sms, T, smem, stream>>>(D1, W);
    XRD_LAUNCH_CHECK();
    XRD_CUDA_TRY(importance(C, cfg, m, L, z, stream));
  }
  {
    KernelTimer kt(stream);
    k_coarse<false><<<gridx, T, smem, stream>>>(D, W);
  }
  XRD_LAUNCH_CHECK();

  XRD_CUDA_TRY(launch_composite<false>(C, stream));
  if (!with_grads) return XRD_OK;

  LossParams LP;
  LP.R = R; LP.is_mapping = 1; LP.with_color = 0; LP.handle_dynamic = 0; LP.use_color_in_tracking = 0;
  LP.w_color = 0.f; LP.target_s = rays->target_s; LP.target_d = rays->target_d;
  LP.rgb = out->rgb; LP.depth = out->depth; LP.var = out->uncertainty;
  LP.gd = L.gd; LP.gc = L.gc;
  LP.tmp = L.tmp; LP.losses = out->losses;
  k_loss<<<1, 1024, 0, stream>>>(LP);
  XRD_LAUNCH_CHECK();
  C.gd = LP.gd; C.gc = LP.gc;
  C.d_occ = L.d_occ;
  XRD_CUDA_TRY(launch_composite<true>(C, stream));
  XRD_CUDA_TRY(cudaMemsetAsync(L.dp, 0, 3 * (size_t)P * 4, stream));
  D.dout[0] = C.d_occ;
  XRD_CUDA_TRY(cudaFuncSetAttribute(k_coarse<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_coarse<true><<<gridx, T, smem, stream>>>(D, W);
  XRD_LAUNCH_CHECK();
  if (d_rays_o || d_rays_d) {
    k_rayreduce<<<(R + 3) / 4, 128, 0, stream>>>(R, S, P, z, L.dp, d_rays_o, d_rays_d);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}
