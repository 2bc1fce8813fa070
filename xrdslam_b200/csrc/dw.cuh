// Generic weight-gradient kernel shared by the per-point MLP pipelines (NICE-SLAM, Vox-Fusion,
// Point-SLAM): activations and their gradients live in HBM in [feature][point] order; a job
// accumulates  out[j*sj + i*si] += sum_p B_j[p] * A_i[p]  (and bias[j] += sum_p B_j[p]) with a
// shared-memory tiled GEMM over a chunk of points per CTA and red.global.add at the end.
//   k_dw_tc (default): tensor cores, mma.sync m16n8k8 TF32 with the 3xTF32 split (fp32-level
//            accuracy): both operands are K-major as they lie in HBM (K = points), so the
//            fragments come straight out of the staged [row][64 points] tiles, conflict-free
//            with a row pitch of 68 floats.  32 x 128 outputs per CTA, 8 warps x (2 x 2) tiles.
//   k_dw    (xrd_debug_gemm_mode 0): the fp32 SIMT reference version.
#pragma once
#include "common.cuh"

namespace xrd {
extern thread_local int g_gemm_mode;  // cabi.cu (0 SIMT, 1 default, 2 TF32, 3 3xTF32 mma.sync)
// out[j*sj + i*si] += sum_p Brow_j[p] (masked) * Arow_i[p];  bias[j] += sum_p Brow_j[p] (masked)
struct DwJob {
  const float* A; int nA;          // rows of Pp floats
  const float* B; int nB;
  const uint32_t* mask;            // per-point relu mask word (bit j) or NULL
  float* out; int sj, si;
  float* bias;                     // or NULL
};
constexpr int DW_MAX_JOBS = 32;
struct DwParams {
  DwJob jobs[DW_MAX_JOBS];
  int n_jobs, P, Pp, chunk;
};

static __global__ void __launch_bounds__(256) k_dw(const DwParams Q) {
  __shared__ float As[128][65];
  __shared__ float Bs[32][65];
  const int tid = threadIdx.x, ta = tid >> 3, tb = tid & 7;
  const int p_lo = blockIdx.x * Q.chunk, p_hi = min(Q.P, p_lo + Q.chunk);
  if (p_lo >= p_hi) return;
  {  // one (chunk of points, job) pair per CTA: grid = (chunks, n_jobs)
    const DwJob J = Q.jobs[blockIdx.y];
    const int nA_it = J.nA > 0 ? J.nA : (J.bias ? 1 : 0);  // bias-only jobs (nA = 0) still sum B
    for (int a0 = 0; a0 < nA_it; a0 += 128) {
      const int na = max(0, min(128, J.nA - a0));
      float acc[4][4];
      float bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      for (int p0 = p_lo; p0 < p_hi; p0 += 64) {
        const int np = min(64, p_hi - p0);
        __syncthreads();
        for (int q = tid; q < 128 * 64; q += 256) {
          const int row = q >> 6, pp = q & 63;
          As[row][pp] = (row < na && pp < np) ? J.A[(size_t)(a0 + row) * Q.Pp + p0 + pp] : 0.f;
        }
        for (int q = tid; q < 32 * 64; q += 256) {
          const int row = q >> 6, pp = q & 63;
          float v = 0.f;
          if (row < J.nB && pp < np) {
            v = J.B[(size_t)row * Q.Pp + p0 + pp];
            if (J.mask && !((J.mask[p0 + pp] >> row) & 1u)) v = 0.f;
          }
          Bs[row][pp] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int pp = 0; pp < 64; ++pp) {
          float av[4], bv[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) av[i] = As[4 * ta + i][pp];
#pragma unroll
          for (int j = 0; j < 4; ++j) bv[j] = Bs[4 * tb + j][pp];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
          if (ta == 0)
#pragma unroll
            for (int j = 0; j < 4; ++j) bacc[j] += bv[j];
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ia = a0 + 4 * ta + i, jbk = 4 * tb + j;
          if (4 * ta + i < na && jbk < J.nB && acc[i][j] != 0.f)
            red_add(J.out + (size_t)jbk * J.sj + (size_t)ia * J.si, acc[i][j]);
        }
      if (ta == 0 && a0 == 0 && J.bias)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (4 * tb + j < J.nB) red_add(J.bias + 4 * tb + j, bacc[j]);
    }
  }
}

// ---- tensor-core version --------------------------------------------------------------------
// Jobs that share their A rows (the 32-row slices of one weight matrix) are merged into a GROUP of
// up to 128 B rows per CTA: A is then read once per weight matrix instead of once per slice
// (Vox-Fusion: 1.5 GB -> 0.72 GB of activation reads per iteration, the kernel is bound by them).
struct DwGroup {
  const float* A; int nA;
  const float* B; int nB;          // nB <= 128, slices of 32 rows
  const uint32_t* mask[4];         // relu mask words of each 32-row slice (bit = row & 31) or NULL
  float* out; int sj, si;
  float* bias;
};
struct DwGParams {
  DwGroup g[DW_MAX_JOBS];
  int n_groups, P, Pp, chunk;
};

__device__ __forceinline__ void dw_mma(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
constexpr int DW_LD = 68;  // floats per staged row: 64 points + 4 (== 4 mod 32: conflict-free fragments)
constexpr int DW_SMEM = 2 * 128 * DW_LD * 4;

// CTA = (chunk of points, group): out[128 x 128] += B[128 x pts] A[128 x pts]^T; 8 warps as 4 (M: 32 B
// rows) x 2 (N: 64 A rows), 2 x 8 m16n8k8 tiles each; 3xTF32 (PREC3) keeps fp32-level accuracy.
template <bool PREC3>
static __global__ void __launch_bounds__(256, 2) k_dw_tc(const DwGParams Q) {
  extern __shared__ __align__(16) float dw_sm[];
  float* As = dw_sm;                  // [128][DW_LD] rows of A (the MMA N side)
  float* Bs = dw_sm + 128 * DW_LD;    // [128][DW_LD] rows of B (the MMA M side), relu-masked
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const int p_lo = blockIdx.x * Q.chunk, p_hi = min(Q.P, p_lo + Q.chunk);
  if (p_lo >= p_hi) return;
  const DwGroup& J = Q.g[blockIdx.y];
  const bool vec = ((Q.Pp & 3) == 0) && ((((uintptr_t)J.A) & 15) == 0) && ((((uintptr_t)J.B) & 15) == 0);
  const bool m_on = wm * 32 < J.nB;
  const int nA_it = J.nA > 0 ? J.nA : (J.bias ? 1 : 0);  // bias-only jobs (nA = 0) still sum B
  for (int a0 = 0; a0 < nA_it; a0 += 128) {
    const int na = max(0, min(128, J.nA - a0));
    const int ntc = max(0, min(8, (na - wn * 64 + 7) / 8));  // live n-tiles of this warp
    float acc[2][8][4];
    float bacc = 0.f;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
    for (int p0 = p_lo; p0 < p_hi; p0 += 64) {
      __syncthreads();
      // stage 128 rows of A and 128 rows of B, 64 points each (16 float4 per row), 8 loads in flight
#pragma unroll
      for (int q0 = 0; q0 < 16; q0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = tid + (q0 + u) * 256;    // 0..2047: A, 2048..4095: B
          const bool isB = e >= 2048;
          const int row = (e & 2047) >> 4;
          const int c4 = (e & 15) * 4, pp = p0 + c4;
          const bool row_ok = isB ? row < J.nB : row < na;
          v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (row_ok && pp < p_hi) {
            const float* src = (isB ? J.B + (size_t)row * Q.Pp : J.A + (size_t)(a0 + row) * Q.Pp) + pp;
            if (vec && pp + 3 < p_hi) {
              v[u] = *reinterpret_cast<const float4*>(src);
            } else {
              v[u].x = src[0];
              if (pp + 1 < p_hi) v[u].y = src[1];
              if (pp + 2 < p_hi) v[u].z = src[2];
              if (pp + 3 < p_hi) v[u].w = src[3];
            }
            const uint32_t* mk = isB ? J.mask[row >> 5] : nullptr;
            if (mk) {
              const int bit = row & 31;
              if (!((mk[pp] >> bit) & 1u)) v[u].x = 0.f;
              if (pp + 1 < p_hi && !((mk[pp + 1] >> bit) & 1u)) v[u].y = 0.f;
              if (pp + 2 < p_hi && !((mk[pp + 2] >> bit) & 1u)) v[u].z = 0.f;
              if (pp + 3 < p_hi && !((mk[pp + 3] >> bit) & 1u)) v[u].w = 0.f;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = tid + (q0 + u) * 256;
          const int row = (e & 2047) >> 4, c4 = (e & 15) * 4;
          *reinterpret_cast<float4*>((e >= 2048 ? Bs : As) + row * DW_LD + c4) = v[u];
        }
      }
      __syncthreads();
      if (a0 == 0 && J.bias) {  // thread = (B row, half of the 64 points)
        const float4* b4 = reinterpret_cast<const float4*>(Bs + (tid >> 1) * DW_LD + (tid & 1) * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 x = b4[i];
          bacc += (x.x + x.y) + (x.z + x.w);
        }
      }
      if (!m_on || ntc == 0) continue;
#pragma unroll 1
      for (int ks = 0; ks < 64; ks += 8) {
        uint32_t ab[2][4], as_[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const float* a = Bs + (wm * 32 + mt * 16 + g) * DW_LD + ks + t;
          const float av[4] = {a[0], a[8 * DW_LD], a[4], a[8 * DW_LD + 4]};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (PREC3) {
              ab[mt][i] = __float_as_uint(av[i]) & 0xffffe000u;
              as_[mt][i] = __float_as_uint(av[i] - __uint_as_float(ab[mt][i]));
            } else {
              ab[mt][i] = __float_as_uint(av[i]);
            }
          }
        }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          if (nt < ntc) {
            const float* b = As + (wn * 64 + nt * 8 + g) * DW_LD + ks + t;
            const float v0 = b[0], v1 = b[4];
            uint32_t bb[2], bs[2];
            if (PREC3) {
              bb[0] = __float_as_uint(v0) & 0xffffe000u;
              bb[1] = __float_as_uint(v1) & 0xffffe000u;
              bs[0] = __float_as_uint(v0 - __uint_as_float(bb[0]));
              bs[1] = __float_as_uint(v1 - __uint_as_float(bb[1]));
            } else {
              bb[0] = __float_as_uint(v0); bb[1] = __float_as_uint(v1);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              if (PREC3) {
                dw_mma(acc[mt][nt], as_[mt], bb);
                dw_mma(acc[mt][nt], ab[mt], bs);
              }
              dw_mma(acc[mt][nt], ab[mt], bb);
            }
          }
        }
      }
    }
    if (m_on) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int j = wm * 32 + mt * 16 + g + ((i & 2) ? 8 : 0);
            const int col = wn * 64 + nt * 8 + 2 * t + (i & 1);
            const float v = acc[mt][nt][i];
            if (nt < ntc && j < J.nB && col < na && v != 0.f)
              red_add(J.out + (size_t)j * J.sj + (size_t)(a0 + col) * J.si, v);
          }
    }
    if (a0 == 0 && J.bias) {
      const float sum = bacc + __shfl_xor_sync(0xffffffffu, bacc, 1);
      if ((tid & 1) == 0 && (tid >> 1) < J.nB) red_add(J.bias + (tid >> 1), sum);
    }
  }
}

// merge the 32-row jobs of one weight matrix (same A rows, consecutive B rows / output rows /
// bias entries) into groups of up to 128 rows
static inline void dw_build_groups(const DwParams& Q, DwGParams& G) {
  G.n_groups = 0; G.P = Q.P; G.Pp = Q.Pp; G.chunk = Q.chunk;
  bool used[DW_MAX_JOBS] = {false};
  for (int i = 0; i < Q.n_jobs; ++i) {
    if (used[i]) continue;
    used[i] = true;
    const DwJob& J = Q.jobs[i];
    DwGroup& g = G.g[G.n_groups++];
    g.A = J.A; g.nA = J.nA; g.B = J.B; g.nB = J.nB; g.out = J.out; g.sj = J.sj; g.si = J.si; g.bias = J.bias;
    g.mask[0] = J.mask; g.mask[1] = g.mask[2] = g.mask[3] = nullptr;
    bool grew = true;
    while (grew && g.nB % 32 == 0 && g.nB < 128) {
      grew = false;
      for (int k = 0; k < Q.n_jobs; ++k) {
        if (used[k]) continue;
        const DwJob& K = Q.jobs[k];
        const bool bias_ok = (!g.bias && !K.bias) || (g.bias && K.bias == g.bias + g.nB);
        if (K.A == g.A && K.nA == g.nA && K.sj == g.sj && K.si == g.si && K.nB <= 32 &&
            K.B == g.B + (size_t)g.nB * Q.Pp && K.out == g.out + (size_t)g.nB * g.sj && bias_ok) {
          g.mask[g.nB / 32] = K.mask;
          g.nB += K.nB;
          used[k] = true;
          grew = true;
          break;
        }
      }
    }
  }
}

// chunk: as many points per CTA as still give >= ~4 CTAs per SM over (chunks x jobs); a
// multiple of the 64-point staging tile.  Fewer, longer chunks mean fewer red.global.add.
static inline cudaError_t launch_dw(DwParams& Q, cudaStream_t stream) {
  if (Q.n_jobs <= 0 || Q.P <= 0) return cudaSuccess;
  if (g_gemm_mode != 0) {
    // tensor-core path: one wave of (chunk, group) CTAs, 2 resident per SM
    DwGParams G;
    dw_build_groups(Q, G);
    const long long want = 2LL * num_sms();
    long long chunks = (want + G.n_groups - 1) / G.n_groups;
    long long chunk = ((long long)Q.P + chunks - 1) / chunks;
    chunk = (chunk + 63) / 64 * 64;
    if (chunk < 256) chunk = 256;
    G.chunk = (int)chunk;
    dim3 grid((unsigned)((Q.P + G.chunk - 1) / G.chunk), (unsigned)G.n_groups);
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(k_dw_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM);
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(k_dw_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM);
      if (e != cudaSuccess) return e;
      attr_set = true;
    }
    if (g_gemm_mode == 2) k_dw_tc<false><<<grid, 256, DW_SMEM, stream>>>(G);
    else k_dw_tc<true><<<grid, 256, DW_SMEM, stream>>>(G);
    return cudaGetLastError();
  }
  const long long want = 4LL * num_sms();
  long long chunks = (want + Q.n_jobs - 1) / Q.n_jobs;
  if (chunks < 1) chunks = 1;
  long long chunk = ((long long)Q.P + chunks - 1) / chunks;
  chunk = (chunk + 63) / 64 * 64;
  if (chunk < 128) chunk = 128;
  if (chunk > 4096) chunk = 4096;
  Q.chunk = (int)chunk;
  dim3 grid((unsigned)((Q.P + Q.chunk - 1) / Q.chunk), (unsigned)Q.n_jobs);
  k_dw<<<grid, 256, 0, stream>>>(Q);
  return cudaGetLastError();
}

}  // namespace xrd
