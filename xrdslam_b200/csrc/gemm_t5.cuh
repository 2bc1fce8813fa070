// Hopper-native GEMM for the wide per-point MLP layers (Vox-Fusion decoder 16-128-128-129 /
// 144-128-3, Point-SLAM colour trunk 5 x 128): wgmma.mma_async m64n128k8 tf32 with fp32
// accumulators in registers, activation tiles fetched by TMA (cp.async.bulk.tensor) into a
// multi-stage mbarrier pipeline, 3xTF32 error compensation for fp32-level parity.
//
//   C[m][n] = epi( sum_k A(m,k) * B[k][n] )      (same contract as gemm.cuh: k_gemm / k_gemm_tc)
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
#pragma once
#include <cuda.h>

#include "gemm.cuh"

namespace xrd {
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

extern thread_local int g_t5_variant;

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

static inline cudaError_t launch_gemm(const GemmArgs& G, cudaStream_t stream) {
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

}  // namespace xrd
