// Shared device/host helpers for the xrdslam_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "xrdslam_b200.h"

namespace xrd {

extern thread_local int g_last_cuda_error;
extern thread_local cudaEvent_t g_ev_start, g_ev_stop;

// bracket the dominant kernel with the caller's events (xrd_debug_kernel_events)
struct KernelTimer {
  cudaStream_t s;
  explicit KernelTimer(cudaStream_t stream) : s(stream) {
    if (g_ev_start && g_ev_stop) cudaEventRecord(g_ev_start, s);
  }
  ~KernelTimer() {
    if (g_ev_start && g_ev_stop) cudaEventRecord(g_ev_stop, s);
  }
};

inline int cuda_fail(cudaError_t e) {
  g_last_cuda_error = (int)e;
  return XRD_E_CUDA;
}

#define XRD_CUDA_TRY(expr)                          \
  do {                                              \
    cudaError_t _e = (expr);                        \
    if (_e != cudaSuccess) return xrd::cuda_fail(_e); \
  } while (0)

#define XRD_LAUNCH_CHECK() XRD_CUDA_TRY(cudaGetLastError())

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int num_sms();

// ---------------------------------------------------------------- device ---
#ifdef __CUDACC__

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_min_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Vectorised fire-and-forget reduction of one 2-feature entry (sm_90+ PTX).
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b)
               : "memory");
}
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c,
                                           float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a),
               "f"(b), "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ void red_add(float* addr, float a) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(a) : "memory");
}

__device__ __forceinline__ float sigmoidf_acc(float x) {
  return 1.0f / (1.0f + expf(-x));
}

// Philox4x32-10, counter = (idx, 0, 0, 0), key = seed.  Returns 4 uniforms.
__device__ __forceinline__ void philox4(uint64_t seed, uint64_t idx, float out[4]) {
  uint32_t c0 = (uint32_t)idx, c1 = (uint32_t)(idx >> 32), c2 = 0, c3 = 0;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  const float s = 2.3283064365386963e-10f;  // 2^-32
  out[0] = (c0 + 0.5f) * s * 0.99999994f;
  out[1] = (c1 + 0.5f) * s * 0.99999994f;
  out[2] = (c2 + 0.5f) * s * 0.99999994f;
  out[3] = (c3 + 0.5f) * s * 0.99999994f;
}

#endif  // __CUDACC__
}  // namespace xrd
