// Host-side utilities of the C-ABI: version, device check, torch.linspace restatement, tcnn
// hash-grid level layout, and the scan-totals copy shared by the compaction entry points.
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace xrd {
thread_local int g_last_cuda_error = 0;
thread_local cudaEvent_t g_ev_start = nullptr, g_ev_stop = nullptr;

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

__global__ void k_copy_totals(int32_t* counts, const int* a, const int* b) {
  counts[0] = *a;
  if (b) counts[1] = *b;
}

int copy_totals(int32_t* counts, const int* a, const int* b, cudaStream_t stream) {
  k_copy_totals<<<1, 1, 0, stream>>>(counts, a, b);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
}  // namespace xrd

extern "C" int xrd_abi_version(void) { return XRD_ABI_VERSION; }

extern "C" int xrd_last_cuda_error(void) { return xrd::g_last_cuda_error; }

extern "C" int xrd_debug_kernel_events(void* start_event, void* stop_event) {
  xrd::g_ev_start = (cudaEvent_t)start_event;
  xrd::g_ev_stop = (cudaEvent_t)stop_event;
  return XRD_OK;
}

extern "C" int xrd_check_device(int dev) {
  int major = 0;
  cudaError_t e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e != cudaSuccess) return xrd::cuda_fail(e);
  int minor = 0;
  e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (e != cudaSuccess) return xrd::cuda_fail(e);
  return (major == 9 && minor == 0) ? XRD_OK : XRD_E_ARCH;
}

// ATen's CPU linspace (aten/src/ATen/native/cpu/RangeFactoriesKernel.cpp): float step,
// first half counts up from start, second half counts down from end.
extern "C" int xrd_linspace_f32(float start, float end, int steps, float* out) {
  if (!out) return XRD_E_NULL;
  if (steps < 0) return XRD_E_SHAPE;
  if (steps == 0) return XRD_OK;
  if (steps == 1) { out[0] = start; return XRD_OK; }
  const float step = (end - start) / (float)(steps - 1);
  const int halfway = steps / 2;
  for (int i = 0; i < steps; ++i) {
    volatile float prod;
    if (i < halfway) { prod = step * (float)i; out[i] = start + prod; }
    else { prod = step * (float)(steps - i - 1); out[i] = end - prod; }
  }
  return XRD_OK;
}

// tcnn GridEncodingTemplated constructor + grid_scale / grid_resolution.
extern "C" int xrd_hashgrid_layout(XrdHashGrid* g, int n_levels, int log2_hashmap_size,
                                   int base_resolution, float per_level_scale) {
  if (!g) return XRD_E_NULL;
  if (n_levels < 1 || n_levels > XRD_MAX_LEVELS || log2_hashmap_size < 3 || log2_hashmap_size > 30)
    return XRD_E_SHAPE;
  const float log2_pls = log2f(per_level_scale);
  uint32_t offset = 0;
  for (int l = 0; l < XRD_MAX_LEVELS; ++l) {
    g->scale[l] = 0.f; g->resolution[l] = 1; g->size[l] = 0; g->offset[l] = offset; g->hashed[l] = 0;
  }
  for (int l = 0; l < n_levels; ++l) {
    volatile float e = exp2f((float)l * log2_pls);
    volatile float m = e * (float)base_resolution;
    const float scale = m - 1.0f;
    const uint32_t res = (uint32_t)ceilf(scale) + 1u;
    const uint32_t max_params = 0xFFFFFFFFu / 2;
    uint64_t dense = (uint64_t)res * res * res;
    uint32_t n = (powf((float)res, 3.f) > (float)max_params) ? max_params : (uint32_t)dense;
    n = (n + 7u) / 8u * 8u;
    const uint32_t cap = 1u << log2_hashmap_size;
    if (n > cap) n = cap;
    // replay grid_index's stride walk: hashed iff size < stride after the walk
    uint64_t stride = 1;
    for (int d = 0; d < 3 && stride <= n; ++d) stride *= res;
    g->scale[l] = scale; g->resolution[l] = res; g->size[l] = n; g->offset[l] = offset;
    g->hashed[l] = (n < stride) ? 1u : 0u;
    // the kernels' dense path assumes the walk covered all 3 dims
    if (!g->hashed[l] && (uint64_t)res * res > n) return XRD_E_SHAPE;
    offset += n;
  }
  g->n_levels = n_levels;
  g->n_entries = offset;
  return XRD_OK;
}
