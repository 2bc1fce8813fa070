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

// blocks of `threads` threads that cover n items
inline unsigned blocks(long long n, int threads = 256) { return (unsigned)((n + threads - 1) / threads); }

int num_sms();

// counts[0] = *a and, if b is not null, counts[1] = *b, in one launch on stream: copies the totals
// at the end of exclusive scans to the caller.
int copy_totals(int32_t* counts, const int* a, const int* b, cudaStream_t stream);

// cub temp storage carved from a workspace, as the cub call takes it
struct CubTemp { void* ptr; size_t bytes; };

// Carves a caller-owned workspace into typed arrays, each starting on a 256-byte boundary.  A
// workspace layout derives from it and takes its arrays in member initialisers, so the declaration
// order is the layout.  With a null base the pointers are null and only the bytes are counted, so
// the same layout sizes the workspace (xrd_*_workspace_bytes) and carves it (the entry point).
class Carver {
 public:
  // bytes the layout needs; 0 if a cub query failed
  size_t bytes() const { return err_ == cudaSuccess ? used_ : 0; }
  // XRD_OK if the layout fits in workspace_bytes
  int check(size_t workspace_bytes) const {
    if (err_ != cudaSuccess) return cuda_fail(err_);
    return workspace_bytes < used_ ? XRD_E_WORKSPACE : XRD_OK;
  }

 protected:
  explicit Carver(void* base) : base_(static_cast<char*>(base)) {}
  // n elements of T, padded to a multiple of 256 bytes
  template <class T> T* take(size_t n) { return at<T>(align_up(n * sizeof(T), 256)); }
  // n elements of T that end the workspace: no padding after them
  template <class T> T* take_last(size_t n) { return at<T>(n * sizeof(T)); }
  // Temp storage for the largest of several cub algorithms, each sized by a callable
  // cudaError_t(size_t& bytes) that runs it with a null temp pointer.  A failed query leaves the
  // layout unsizable.
  template <class... Q> CubTemp cub(Q... queries) {
    size_t bytes = 0;
    auto query = [&](auto& q) {
      size_t b = 0;
      if (const cudaError_t e = q(b)) err_ = e;
      if (b > bytes) bytes = b;
    };
    (query(queries), ...);
    return {take<char>(bytes), bytes};
  }

 private:
  // the next `bytes` of the workspace as a T*
  template <class T> T* at(size_t bytes) {
    const size_t off = used_;
    used_ += bytes;
    return base_ ? reinterpret_cast<T*>(base_ + off) : nullptr;
  }
  char* base_;
  size_t used_ = 0;
  cudaError_t err_ = cudaSuccess;
};

// ---------------------------------------------------------------- device ---
#ifdef __CUDACC__

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
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
