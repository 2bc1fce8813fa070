// Generic fp32 SIMT GEMM on [feature][point] activations (points contiguous), used by the
// wide per-point MLPs whose layers are real GEMMs (Point-SLAM colour decoder: 128-wide trunk
// over R*5 points and the per-neighbour MLP over 8x as many columns):
//   C[m][n] = epi( sum_k A(m,k) * B[k][n] ),   A(m,k) = transA ? A[k*lda+m] : A[m*lda+k]
//   epi(v)  = act(v + bias[m]);  zeroed where relu_mask[m][n] <= 0 (optional: backward of a
//             relu layer);  act_out[m][n] = epi(v) (optional);  + addend[m][n] (optional);
//             accumulate: C += that.
// 64 x 128 tile, BK = 16, 256 threads, 4 x 8 register tile per thread, fp32 FMA (exact-order
// independent of the tile position, so results do not depend on how points are batched).
#pragma once
#include "common.cuh"

namespace xrd {

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_SOFTPLUS100 = 2, ACT_SIGMOID = 3 };

struct GemmArgs {
  int M, N, K;
  const float* A; int lda; int transA;
  const float* B; int ldb;
  float* C; int ldc;
  const float* bias;
  int act;
  const float* addend; int ldadd;
  float* act_out; int ldact;
  int accumulate;
  const float* relu_mask; int ldmask;  // optional: result zeroed where relu_mask[m][n] <= 0
};

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_SOFTPLUS100: return (v * 100.f > 20.f) ? v : log1pf(expf(v * 100.f)) / 100.f;  // nn.Softplus(beta=100)
    case ACT_SIGMOID: return sigmoidf_acc(v);
    default: return v;
  }
}

constexpr int GBM = 64, GBN = 128, GBK = 16;

static __global__ void __launch_bounds__(256) k_gemm(const GemmArgs G) {
  __shared__ __align__(16) float As[GBK][GBM + 4];
  __shared__ __align__(16) float Bs[GBK][GBN + 4];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const bool b_vec = ((G.ldb & 3) == 0) && ((((uintptr_t)G.B) & 15) == 0);
  for (int k0 = 0; k0 < G.K; k0 += GBK) {
    // A tile: 64 x 16
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int e = tid + q * 256;
      int m, k;
      if (G.transA) { k = e >> 6; m = e & 63; } else { m = e >> 4; k = e & 15; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < G.M && gk < G.K) v = G.transA ? G.A[(size_t)gk * G.lda + gm] : G.A[(size_t)gm * G.lda + gk];
      As[k][m] = v;
    }
    // B tile: 16 x 128 (two float4 per thread)
    {
      const int k = tid >> 4, c = (tid & 15) * 8;
      const int gk = k0 + k;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gn = n0 + c + 4 * h;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gk < G.K) {
          const float* src = G.B + (size_t)gk * G.ldb + gn;
          if (b_vec && gn + 3 < G.N) {
            v = *reinterpret_cast<const float4*>(src);
          } else {
            if (gn < G.N) v.x = src[0];
            if (gn + 1 < G.N) v.y = src[1];
            if (gn + 2 < G.N) v.z = src[2];
            if (gn + 3 < G.N) v.w = src[3];
          }
        }
        *reinterpret_cast<float4*>(&Bs[k][c + 4 * h]) = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GBK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][64 + tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= G.M) continue;
    const float bias = G.bias ? G.bias[gm] : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (gn >= G.N) continue;
      float v = act_apply(acc[i][j] + bias, G.act);
      if (G.relu_mask && !(G.relu_mask[(size_t)gm * G.ldmask + gn] > 0.f)) v = 0.f;
      if (G.act_out) G.act_out[(size_t)gm * G.ldact + gn] = v;
      if (G.addend) v += G.addend[(size_t)gm * G.ldadd + gn];
      float* c = G.C + (size_t)gm * G.ldc + gn;
      *c = G.accumulate ? (*c + v) : v;
    }
  }
}

// ---- tensor-core version: mma.sync.m16n8k8 TF32, optional 3xTF32 split ------------------
// MMA M = output features (A operand = weights, zero-padded to 128 rows in shared memory),
// MMA N = points (B operand = the [K][N] activation rows as they lie in HBM).  128 x 128 x 16
// CTA tile, 8 warps, each warp owns a 16-point slab (2 n-tiles) for all 8 m-tiles: 64 fp32
// accumulators per thread.  Shared-memory strides (20 for A rows, 136 for B rows) make every
// fragment load bank-conflict-free.  3xTF32 (big = x & 0xffffe000, small = x - big;
// a.small*b.big + a.big*b.small + a.big*b.big) keeps fp32-level accuracy (parity tests).
constexpr int TBM = 128, TBN = 128, TBK = 16, TLDA = TBK + 4, TLDB = TBN + 8;

__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4],
                                                const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <bool PREC3>
static __global__ void __launch_bounds__(256, 2) k_gemm_tc(const GemmArgs G) {
  __shared__ __align__(16) float As[TBM * TLDA];
  __shared__ __align__(16) float Bs[TBK * TLDB];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int m0 = blockIdx.y * TBM, n0 = blockIdx.x * TBN;
  const int m_tiles = min(TBM / 16, (G.M - m0 + 15) / 16);
  float acc[TBM / 16][2][4];
#pragma unroll
  for (int mt = 0; mt < TBM / 16; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
  const bool b_vec = ((G.ldb & 3) == 0) && ((((uintptr_t)G.B) & 15) == 0);
  for (int k0 = 0; k0 < G.K; k0 += TBK) {
    // A tile 128 x 16 -> As[m][k]
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int e = tid + q * 256;
      int m, k;
      if (G.transA) { k = e >> 7; m = e & 127; } else { m = e >> 4; k = e & 15; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < G.M && gk < G.K) v = G.transA ? G.A[(size_t)gk * G.lda + gm] : G.A[(size_t)gm * G.lda + gk];
      As[m * TLDA + k] = v;
    }
    // B tile 16 x 128 -> Bs[k][n]
    {
      const int k = tid >> 4, c = (tid & 15) * 8;
      const int gk = k0 + k;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gn = n0 + c + 4 * h;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gk < G.K) {
          const float* src = G.B + (size_t)gk * G.ldb + gn;
          if (b_vec && gn + 3 < G.N) {
            v = *reinterpret_cast<const float4*>(src);
          } else {
            if (gn < G.N) v.x = src[0];
            if (gn + 1 < G.N) v.y = src[1];
            if (gn + 2 < G.N) v.z = src[2];
            if (gn + 3 < G.N) v.w = src[3];
          }
        }
        *reinterpret_cast<float4*>(&Bs[k * TLDB + c + 4 * h]) = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < TBK; ks += 8) {
      uint32_t bb[2][2], bs[2][2];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const int n = warp * 16 + nt * 8 + g;
        const float v0 = Bs[(ks + t) * TLDB + n], v1 = Bs[(ks + t + 4) * TLDB + n];
        if (PREC3) {
          bb[nt][0] = __float_as_uint(v0) & 0xffffe000u;
          bb[nt][1] = __float_as_uint(v1) & 0xffffe000u;
          bs[nt][0] = __float_as_uint(v0 - __uint_as_float(bb[nt][0]));
          bs[nt][1] = __float_as_uint(v1 - __uint_as_float(bb[nt][1]));
        } else {
          bb[nt][0] = __float_as_uint(v0); bb[nt][1] = __float_as_uint(v1);
        }
      }
#pragma unroll
      for (int mt = 0; mt < TBM / 16; ++mt) {
        if (mt >= m_tiles) break;
        const float* a = As + (mt * 16 + g) * TLDA + ks + t;
        const float av[4] = {a[0], a[8 * TLDA], a[4], a[8 * TLDA + 4]};
        uint32_t ab[4], asml[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (PREC3) {
            ab[i] = __float_as_uint(av[i]) & 0xffffe000u;
            asml[i] = __float_as_uint(av[i] - __uint_as_float(ab[i]));
          } else {
            ab[i] = __float_as_uint(av[i]);
          }
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          if (PREC3) {
            mma_tf32_16x8x8(acc[mt][nt], asml, bb[nt]);
            mma_tf32_16x8x8(acc[mt][nt], ab, bs[nt]);
          }
          mma_tf32_16x8x8(acc[mt][nt], ab, bb[nt]);
        }
      }
    }
    __syncthreads();
  }
  // epilogue: c[0],c[1] -> row g, cols 2t, 2t+1 ; c[2],c[3] -> row g+8
#pragma unroll
  for (int mt = 0; mt < TBM / 16; ++mt) {
    if (mt >= m_tiles) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gm = m0 + mt * 16 + g + 8 * h;
      if (gm >= G.M) continue;
      const float bias = G.bias ? G.bias[gm] : 0.f;
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int gn = n0 + warp * 16 + nt * 8 + 2 * t + j;
          if (gn >= G.N) continue;
          float v = act_apply(acc[mt][nt][2 * h + j] + bias, G.act);
          if (G.relu_mask && !(G.relu_mask[(size_t)gm * G.ldmask + gn] > 0.f)) v = 0.f;
          if (G.act_out) G.act_out[(size_t)gm * G.ldact + gn] = v;
          if (G.addend) v += G.addend[(size_t)gm * G.ldadd + gn];
          float* c = G.C + (size_t)gm * G.ldc + gn;
          *c = G.accumulate ? (*c + v) : v;
        }
    }
  }
}

// Arithmetic of the wide-MLP GEMMs (xrd_debug_gemm_mode, cabi.cu):
//   0 = fp32 SIMT (k_gemm)
//   1 = 3xTF32 tensor cores (default): wgmma / TMA kernel (gemm_t5.cuh) for the shapes it
//       takes, mma.sync k_gemm_tc<true> for the rest
//   2 = plain TF32 mma.sync (k_gemm_tc<false>)
//   3 = 3xTF32 mma.sync only (k_gemm_tc<true>; kept for A/B runs)
extern thread_local int g_gemm_mode;

static inline cudaError_t launch_gemm_legacy(const GemmArgs& G, cudaStream_t stream) {
  if (G.M <= 0 || G.N <= 0) return cudaSuccess;
  if (g_gemm_mode == 0 || G.K < 8) {
    dim3 grid((G.N + GBN - 1) / GBN, (G.M + GBM - 1) / GBM);
    k_gemm<<<grid, 256, 0, stream>>>(G);
  } else {
    dim3 grid((G.N + TBN - 1) / TBN, (G.M + TBM - 1) / TBM);
    if (g_gemm_mode != 2) k_gemm_tc<true><<<grid, 256, 0, stream>>>(G);
    else k_gemm_tc<false><<<grid, 256, 0, stream>>>(G);
  }
  return cudaGetLastError();
}

}  // namespace xrd
