// Wide-MLP GEMM and weight-gradient kernels (mlp.cuh), their launchers and the debug entry
// points that run them directly.
#include <cuda.h>

#include "mlp.cuh"

namespace xrd {

// arithmetic of the GEMMs and weight gradients, per calling thread (xrd_debug_gemm_mode)
thread_local int g_gemm_mode = 1;

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_SOFTPLUS100: return (v * 100.f > 20.f) ? v : log1pf(expf(v * 100.f)) / 100.f;  // nn.Softplus(beta=100)
    case ACT_SIGMOID: return sigmoidf_acc(v);
    default: return v;
  }
}

// ---- fp32 SIMT GEMM ---------------------------------------------------------------------
// 64 x 128 tile, BK = 16, 256 threads, 4 x 8 register tile per thread, fp32 FMA (exact-order
// independent of the tile position, so results do not depend on how points are batched).
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

// ---- Hopper-native GEMM -------------------------------------------------------------------
// For the wide per-point MLP layers (Vox-Fusion decoder 16-128-128-129 / 144-128-3, Point-SLAM
// colour trunk 5 x 128), same contract as k_gemm / k_gemm_tc: wgmma.mma_async m64n128k8 tf32
// with fp32 accumulators in registers, activation tiles fetched by TMA (cp.async.bulk.tensor)
// into a multi-stage mbarrier pipeline, 3xTF32 error compensation for fp32-level parity.
//
// wgmma takes tf32 operands from shared memory only K-major, and the activations lie in HBM
// points-contiguous ([K][N]), so the roles are swapped against the math:
//   MMA M = points (64 per consumer warpgroup, 128 per tile), the A operand from REGISTERS:
//      every thread reads its fragment straight out of the raw TMA tile (BK rows x BP points,
//      row-major) and splits it into big = x with the 13 low mantissa bits cleared and
//      small = x - big;
//   MMA N = 128 output features (the weights, zero padded), the B operand from SHARED memory,
//      staged ONCE per CTA by all threads (handles transA / lda / padding) as big / small in the
//      canonical no-swizzle K-major layout (core matrix = 8 rows x 16 bytes):
//      off(row, k) = (k/4) * (NF*16) + row*16 + (k%4)*4      LBO = NF*16 B (K), SBO = 128 B (rows)
//   D: 64 fp32 registers per thread (m64n128), so the epilogue writes C[feature][point] with
//      the 8 lanes of a quad group covering 8 consecutive points (full 32-byte sectors).
// Roles (288 threads): warps 0-7 = two consumer warpgroups (fragment loads, 3 wgmma per k8
// step, epilogue), warp 8 = TMA producer (one elected lane).  The producer runs up to STAGES
// k-blocks ahead, across tile boundaries, so the next tile's loads overlap this tile's epilogue.
// All hand-offs are mbarriers; every wait is bounded (a broken pipeline traps instead of
// hanging the GPU).

namespace t5 {

constexpr int NF = 128;  // output features per launch (the wgmma N)
constexpr int BM = NF;   // rows of C one launch covers (launch_gemm splits taller GEMMs)
constexpr int BP = 128;  // points per tile: 2 consumer warpgroups x 64
constexpr int BK = 16;   // k rows per pipeline stage (2 wgmma k-steps)
constexpr int STAGES = 4;
constexpr int NTHREADS = 288;
constexpr uint32_t SPIN_LIMIT = 1u << 27;

struct Params {
  GemmArgs G;
  int Kpad;      // K rounded up to BK
  int n_tiles;   // ceil(N / BP)
  int variant;   // debug (xrd_debug_gemm_variant): bit 0 swaps LBO / SBO in the descriptors
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t done = 0, spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(a), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins > SPIN_LIMIT) __trap();  // broken pipeline: fail loudly, never hang
  }
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 points][128 features] (+)= A[64 points][8 k] (registers) * B[8 k][128 features] (smem)
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b,
                                           uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d)
      : "memory");
}

// shared-memory matrix descriptor (sm_90 GMMA): start address, leading / stride byte offsets
// (16-byte units), base offset 0, layout type 0 (no swizzle) in bits [62,64)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  return d;
}

__device__ __forceinline__ float tf32_big(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

static __global__ void __launch_bounds__(NTHREADS, 1)
k_gemm_t5(const __grid_constant__ CUtensorMap tmap_b, const Params P) {
  constexpr int RAW_BYTES = BK * BP * 4;  // one TMA box: BK rows x BP points, row-major
  extern __shared__ __align__(1024) uint8_t smem[];
  const GemmArgs& G = P.G;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int Kpad = P.Kpad;
  const int w_bytes = NF * Kpad * 4;
  float* w_big = reinterpret_cast<float*>(smem);
  float* w_small = reinterpret_cast<float*>(smem + w_bytes);
  uint8_t* raw_base = smem + 2 * w_bytes;  // [STAGES][RAW_BYTES]
  uint64_t* full = reinterpret_cast<uint64_t*>(raw_base + STAGES * RAW_BYTES);  // [STAGES] TMA bytes landed
  uint64_t* empty = full + STAGES;  // [STAGES] fragments read by all 256 consumer threads

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 256); }
    fence_barrier_init();
  }
  // ---- stage the weights once: A(m,k) -> canonical K-major core-matrix layout, big / small.
  // lane = (m & 7) | (k & 3) << 3: conflict-free shared-memory writes (32 consecutive floats),
  // 8 rows x 16 bytes (row-major A) or 4 rows x 32 bytes (transposed A) per global request;
  // 8 independent loads in flight per thread
  {
    const int n_e = NF * Kpad;
    for (int e0 = tid; e0 < n_e; e0 += NTHREADS * 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = e0 + u * NTHREADS;
        const int hi = e >> 5, lo = e & 31;
        const int m = ((hi % (NF / 8)) << 3) | (lo & 7);
        const int k = ((hi / (NF / 8)) << 2) | (lo >> 3);
        v[u] = 0.f;
        if (e < n_e && m < G.M && k < G.K)
          v[u] = G.transA ? G.A[(size_t)k * G.lda + m] : G.A[(size_t)m * G.lda + k];
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = e0 + u * NTHREADS;
        if (e < n_e) {
          const int hi = e >> 5, lo = e & 31;
          const int m = ((hi % (NF / 8)) << 3) | (lo & 7);
          const int k = ((hi / (NF / 8)) << 2) | (lo >> 3);
          const float big = tf32_big(v[u]);
          const int off = (k >> 2) * (NF * 4) + m * 4 + (k & 3);
          w_big[off] = big;
          w_small[off] = v[u] - big;
        }
      }
    }
  }
  fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
  __syncthreads();
  const int n_kb = Kpad / BK;

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
        for (int kb = 0; kb < n_kb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
          mbar_expect_tx(full + s, RAW_BYTES);
          tma_load_2d(raw_base + (size_t)s * RAW_BYTES, &tmap_b, full + s, tile * BP, kb * BK);
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup c owns points [c*64, c*64 + 64) of a tile ======
  const int c = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
  const int pl = c * 64 + wq * 16 + g;  // this thread's first point in the tile (second: + 8)
  const bool swap = (P.variant & 1) != 0;
  const uint32_t lbo = swap ? 128u : NF * 16u, sbo = swap ? NF * 16u : 128u;
  const uint32_t wb = smem_u32(w_big), ws = smem_u32(w_small);
  int it = 0;
  for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < n_kb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(full + s, (it / STAGES) & 1);
      const float* raw = reinterpret_cast<const float*>(raw_base + (size_t)s * RAW_BYTES);
      // A fragment of m64n128k8 (per warp: 16 points x 8 k): a0 = (g, t), a1 = (g + 8, t),
      // a2 = (g, t + 4), a3 = (g + 8, t + 4) as (point, k)
      uint32_t ab[BK / 8][4], as[BK / 8][4];
#pragma unroll
      for (int ks = 0; ks < BK / 8; ++ks) {
        const float* r0 = raw + (ks * 8 + t) * BP + pl;
        const float* r4 = r0 + 4 * BP;
        const float v[4] = {r0[0], r0[8], r4[0], r4[8]};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float big = tf32_big(v[i]);
          ab[ks][i] = __float_as_uint(big);
          as[ks][i] = __float_as_uint(v[i] - big);
        }
      }
      mbar_arrive(empty + s);  // the raw slot may be refilled
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BK / 8; ++ks) {
        const uint32_t koff = (uint32_t)(kb * (BK / 4) + ks * 2) * (NF * 16);  // 16-byte K chunks
        const uint64_t db = make_desc(wb + koff, lbo, sbo), dsm = make_desc(ws + koff, lbo, sbo);
        wgmma_tf32(acc, as[ks], db, (kb | ks) != 0 ? 1u : 0u);  // small terms first (3xTF32)
        wgmma_tf32(acc, ab[ks], dsm, 1u);
        wgmma_tf32(acc, ab[ks], db, 1u);
      }
      wgmma_commit();
      wgmma_wait_all();  // the A fragments live in registers that the next k-block reuses
    }
    // ---- epilogue: acc[4i + 2h + j] = (point pl + 8h, feature 8i + 2t + j)
    const int n0 = tile * BP + pl;
#pragma unroll
    for (int i = 0; i < NF / 8; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int m = 8 * i + 2 * t + j;
        if (m >= G.M) continue;
        const float bias = G.bias ? G.bias[m] : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = n0 + 8 * h;
          if (n >= G.N) continue;
          float v = act_apply(acc[4 * i + 2 * h + j] + bias, G.act);
          if (G.relu_mask && !(G.relu_mask[(size_t)m * G.ldmask + n] > 0.f)) v = 0.f;
          if (G.act_out) G.act_out[(size_t)m * G.ldact + n] = v;
          if (G.addend) v += G.addend[(size_t)m * G.ldadd + n];
          float* cp = G.C + (size_t)m * G.ldc + n;
          *cp = G.accumulate ? (*cp + v) : v;
        }
      }
    }
  }
}

// ---- host side --------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// shapes this kernel takes (everything else stays on k_gemm_tc / k_gemm)
static inline bool eligible(const GemmArgs& G) {
  return G.M >= 16 && G.M <= BM && G.K >= 16 && G.K <= 144 && G.N >= 512 && (G.ldb & 3) == 0 &&
         ((((uintptr_t)G.B) & 15) == 0) && encode_fn() != nullptr;
}

thread_local int g_t5_variant = 0;  // xrd_debug_gemm_variant

static inline cudaError_t launch(const GemmArgs& G, cudaStream_t stream) {
  Params P;
  P.G = G;
  P.Kpad = (G.K + BK - 1) / BK * BK;
  P.n_tiles = (G.N + BP - 1) / BP;
  P.variant = g_t5_variant;
  // B [K][ldb] fp32 as a 2-D tensor (points innermost); box = (BP points, BK rows), no swizzle;
  // rows >= K and columns >= ldb read as zero (out-of-bounds fill)
  CUtensorMap tm;
  const cuuint64_t dims[2] = {(cuuint64_t)G.ldb, (cuuint64_t)G.K};
  const cuuint64_t strides[1] = {(cuuint64_t)G.ldb * 4};  // bytes, dim 1
  const cuuint32_t box[2] = {BP, BK};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(G.B), dims, strides,
                           box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cudaErrorInvalidValue;
  // resident weights (big + small, 2 x 128 x Kpad x 4 B: 144 KB at K = 144) + STAGES raw
  // activation tiles (8 KB each) + barriers must fit the 227 KB an H100 block may use
  const size_t smem = 2 * (size_t)NF * P.Kpad * 4 + (size_t)STAGES * BK * BP * 4 + 2 * STAGES * 8;
  if (smem > 232448) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_gemm_t5, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  int grid = P.n_tiles < num_sms() ? P.n_tiles : num_sms();
  k_gemm_t5<<<grid, NTHREADS, smem, stream>>>(tm, P);
  return cudaGetLastError();
}

}  // namespace t5

// rows [m0, m0 + mc) of a GEMM as a GEMM of its own
static inline GemmArgs gemm_rows(const GemmArgs& G, int m0, int mc) {
  GemmArgs H = G;
  H.M = mc;
  H.A = G.transA ? G.A + m0 : G.A + (size_t)m0 * G.lda;
  H.C = G.C + (size_t)m0 * G.ldc;
  if (G.bias) H.bias = G.bias + m0;
  if (G.addend) H.addend = G.addend + (size_t)m0 * G.ldadd;
  if (G.act_out) H.act_out = G.act_out + (size_t)m0 * G.ldact;
  if (G.relu_mask) H.relu_mask = G.relu_mask + (size_t)m0 * G.ldmask;
  return H;
}

cudaError_t launch_gemm(const GemmArgs& G, cudaStream_t stream) {
  if (G.M <= 0 || G.N <= 0) return cudaSuccess;
  if (g_gemm_mode == 1) {
    if (t5::eligible(G)) return t5::launch(G, stream);
    if (G.M > t5::BM) {  // e.g. 144 = 128 + 16 rows: two launches
      GemmArgs top = gemm_rows(G, 0, t5::BM);
      if (t5::eligible(top)) {
        cudaError_t e = t5::launch(top, stream);
        if (e != cudaSuccess) return e;
        return launch_gemm(gemm_rows(G, t5::BM, G.M - t5::BM), stream);
      }
    }
  }
  return launch_gemm_legacy(G, stream);
}

// ---- weight gradients -------------------------------------------------------------------
// Shared by the per-point MLP pipelines (NICE-SLAM, Vox-Fusion, Point-SLAM): activations and their gradients live in HBM in [feature][point] order; a job
// accumulates  out[j*sj + i*si] += sum_p B_j[p] * A_i[p]  (and bias[j] += sum_p B_j[p]) with a
// shared-memory tiled GEMM over a chunk of points per CTA and red.global.add at the end.
//   k_dw_tc (default): tensor cores, mma.sync m16n8k8 TF32 with the 3xTF32 split (fp32-level
//            accuracy): both operands are K-major as they lie in HBM (K = points), so the
//            fragments come straight out of the staged [row][64 points] tiles, conflict-free
//            with a row pitch of 68 floats.  32 x 128 outputs per CTA, 8 warps x (2 x 2) tiles.
//   k_dw    (xrd_debug_gemm_mode 0): the fp32 SIMT reference version.

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
cudaError_t launch_dw(DwParams& Q, cudaStream_t stream) {
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

extern "C" int xrd_debug_gemm_mode(int mode) {
  if (mode < 0 || mode > 3) return XRD_E_SHAPE;
  xrd::g_gemm_mode = mode;
  return XRD_OK;
}

extern "C" int xrd_debug_gemm_variant(int variant) {
  xrd::t5::g_t5_variant = variant;
  return XRD_OK;
}

// Direct entry to the wide-MLP GEMM for the unit tests:
//   C[m][n] = act( sum_k A(m,k) B[k][n] + bias[m] ), optional relu mask / addend, under the
//   calling thread's xrd_debug_gemm_mode.  All pointers DEVICE.
extern "C" int xrd_debug_gemm(int M, int N, int K, const float* A, int lda, int transA, const float* B,
                              int ldb, float* C, int ldc, const float* bias, int act,
                              const float* relu_mask, int ldmask, const float* addend, int ldadd,
                              void* stream) {
  if (!A || !B || !C) return XRD_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0) return XRD_E_SHAPE;
  xrd::GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.A = A; g.lda = lda; g.transA = transA; g.B = B; g.ldb = ldb;
  g.C = C; g.ldc = ldc; g.bias = bias; g.act = act; g.relu_mask = relu_mask; g.ldmask = ldmask;
  g.addend = addend; g.ldadd = ldadd;
  XRD_CUDA_TRY(xrd::launch_gemm(g, (cudaStream_t)stream));
  return XRD_OK;
}

// ... with the remaining epilogue options: act_out[m][n] receives the masked activation before
// the addend, accumulate != 0 adds the result to C.
extern "C" int xrd_debug_gemm_ex(int M, int N, int K, const float* A, int lda, int transA, const float* B,
                                 int ldb, float* C, int ldc, const float* bias, int act,
                                 const float* relu_mask, int ldmask, const float* addend, int ldadd,
                                 float* act_out, int ldact, int accumulate, void* stream) {
  if (!A || !B || !C) return XRD_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0) return XRD_E_SHAPE;
  xrd::GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.A = A; g.lda = lda; g.transA = transA; g.B = B; g.ldb = ldb;
  g.C = C; g.ldc = ldc; g.bias = bias; g.act = act; g.relu_mask = relu_mask; g.ldmask = ldmask;
  g.addend = addend; g.ldadd = ldadd; g.act_out = act_out; g.ldact = ldact; g.accumulate = accumulate;
  XRD_CUDA_TRY(xrd::launch_gemm(g, (cudaStream_t)stream));
  return XRD_OK;
}

// Direct entry to the weight-gradient kernels for the unit tests:
//   out[j][i] += sum_p B[j][p] (where bit (j & 31) of mask[j / 32][p] is set) * A[i][p],
//   bias[j] += sum_p B[j][p] (masked)
// A [nA][Pp], B [nB][Pp] rows of P valid points; the rows of B are cut into 32-row jobs exactly
// as the model kernels do, under the calling thread's xrd_debug_gemm_mode.  DEVICE pointers.
extern "C" int xrd_debug_dw(int nA, int nB, int P, int Pp, const float* A, const float* B,
                            const uint32_t* mask, float* out, float* bias, void* stream) {
  if (!A || !B || !out) return XRD_E_NULL;
  if (nA <= 0 || nB <= 0 || P <= 0 || Pp < P) return XRD_E_SHAPE;
  xrd::DwParams D;
  D.n_jobs = 0; D.P = P; D.Pp = Pp; D.chunk = 512;
  for (int c = 0; c < nB; c += 32) {
    if (D.n_jobs >= xrd::DW_MAX_JOBS) return XRD_E_SHAPE;
    xrd::DwJob& J = D.jobs[D.n_jobs++];
    J.A = A; J.nA = nA; J.B = B + (size_t)c * Pp; J.nB = nB - c < 32 ? nB - c : 32;
    J.mask = mask ? mask + (size_t)(c / 32) * P : nullptr;
    J.out = out + (size_t)c * nA; J.sj = nA; J.si = 1;
    J.bias = bias ? bias + c : nullptr;
  }
  XRD_CUDA_TRY(xrd::launch_dw(D, (cudaStream_t)stream));
  return XRD_OK;
}
