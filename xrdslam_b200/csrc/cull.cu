// cull_mesh on the device (sm_90a): which mesh vertices some frame sees, then the faces that
// keep a seen vertex and the vertices those faces reference.
//
// Replaces (reference @ f0366f20):
//   slam/common/common.py:714-789  cull_mesh: per frame an H2D copy of every vertex (float64),
//                                  ~20 torch launches and a D2H copy of the mask, ANDed on the
//                                  host; then trimesh's update_faces /
//                                  remove_unreferenced_vertices
// Semantics (fixed here, documented in include/xrdslam_b200.h): the reference's projection and
// bilinear depth sample in fp32 with explicit round-to-nearest intrinsics in its expression
// order; visibility is an OR over frames, so the result does not depend on how vertices and
// frames are split over threads and launches.  Compaction is order-preserving (two exclusive
// scans), in two phases like xrd_mesh_mc_*.
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace xrd {
namespace cull {

// row r of a [3][4] transform applied to (x, y, z, 1), summed in k order (w * 1 is exact)
__device__ __forceinline__ float row(const float* T, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)),
                             __fmul_rn(T[2], z)),
                   T[3]);
}

// grid_sample(depth, 2 * (u / W, v / H) - 1, bilinear, zeros, align_corners=True) at one point
// that passed the frustum tests (so the source coordinates lie in [0, size - 1])
__device__ __forceinline__ float sample_depth(const float* __restrict__ D, int H, int W, float u,
                                              float v) {
  const float gx = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(u, (float)W)), 1.f);
  const float gy = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(v, (float)H)), 1.f);
  const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(W - 1));
  const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(H - 1));
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f);
  const float nw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(y1, iy));
  const float ne = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(y1, iy));
  const float sw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(iy, y0));
  const float se = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(iy, y0));
  const int c0 = (int)x0, r0 = (int)y0, c1 = c0 + 1, r1 = r0 + 1;
  const bool in_c0 = c0 >= 0 && c0 < W, in_c1 = c1 >= 0 && c1 < W;
  const bool in_r0 = r0 >= 0 && r0 < H, in_r1 = r1 >= 0 && r1 < H;
  float d = 0.f;
  if (in_r0 && in_c0) d = __fadd_rn(d, __fmul_rn(__ldg(D + (size_t)r0 * W + c0), nw));
  if (in_r0 && in_c1) d = __fadd_rn(d, __fmul_rn(__ldg(D + (size_t)r0 * W + c1), ne));
  if (in_r1 && in_c0) d = __fadd_rn(d, __fmul_rn(__ldg(D + (size_t)r1 * W + c0), sw));
  if (in_r1 && in_c1) d = __fadd_rn(d, __fmul_rn(__ldg(D + (size_t)r1 * W + c1), se));
  return d;
}

// one thread per vertex, looping over the launch's frames until one sees it; w2c staged in
// shared memory ([n_frames][12] floats)
__global__ void __launch_bounds__(256) k_cull_visible(const float* __restrict__ verts, int V,
                                                      const float* __restrict__ w2c,
                                                      const float* __restrict__ depth, int F,
                                                      XrdCullParams P,
                                                      uint8_t* __restrict__ seen) {
  extern __shared__ float s_w2c[];
  for (int i = threadIdx.x; i < F * 12; i += blockDim.x) s_w2c[i] = __ldg(w2c + i);
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || seen[v]) return;
  const float x = __ldg(verts + (size_t)v * 3), y = __ldg(verts + (size_t)v * 3 + 1),
              z = __ldg(verts + (size_t)v * 3 + 2);
  const float Wf = (float)P.W, Hf = (float)P.H;
  const size_t plane = (size_t)P.H * P.W;
  for (int f = 0; f < F; ++f) {
    const float* T = s_w2c + 12 * f;
    const float xc = -row(T, x, y, z);  // cam_cord[:, 0] *= -1
    const float yc = row(T + 4, x, y, z);
    const float zc = row(T + 8, x, y, z);
    // K @ cam with K's zero entries left out: a +-0 term changes no decision below
    const float up = __fadd_rn(__fmul_rn(P.fx, xc), __fmul_rn(P.cx, zc));
    const float vp = __fadd_rn(__fmul_rn(P.fy, yc), __fmul_rn(P.cy, zc));
    const float zz = __fadd_rn(zc, 1e-5f);
    const float u = __fdiv_rn(up, zz), vv = __fdiv_rn(vp, zz);
    // frustum first (false for NaN): depth is read only for points inside the image
    if (!(0.f <= -zz) || !(u < Wf) || !(u > 0.f) || !(vv < Hf) || !(vv > 0.f)) continue;
    if (P.eval_rec) {
      const float d = sample_depth(depth + plane * f, P.H, P.W, u, vv);
      if (!(__fadd_rn(d, P.truncation) >= -zz)) continue;
    }
    seen[v] = 1;
    return;
  }
}

// per face: keep flag (some vertex seen), and reference flags for the vertices of kept faces;
// faces with an index outside [0, V) are counted in *bad and neither kept nor dereferenced
__global__ void __launch_bounds__(256) k_cull_faces(const uint8_t* __restrict__ seen, int V,
                                                    const int32_t* __restrict__ faces, int Fn,
                                                    int* __restrict__ keep, int* __restrict__ ref,
                                                    int32_t* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > Fn) return;
  if (f == Fn) { keep[f] = 0; return; }
  int id[3];
  bool ok = true;
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    id[m] = __ldg(faces + (size_t)f * 3 + m);
    ok = ok && id[m] >= 0 && id[m] < V;
  }
  if (!ok) {
    keep[f] = 0;
    atomicAdd(bad, 1);
    return;
  }
  const int k = (seen[id[0]] | seen[id[1]] | seen[id[2]]) ? 1 : 0;
  keep[f] = k;
  if (k) ref[id[0]] = ref[id[1]] = ref[id[2]] = 1;  // same value from every writer
}

__global__ void __launch_bounds__(256) k_cull_emit_verts(const float* __restrict__ verts,
                                                         const uint8_t* __restrict__ colors,
                                                         int color_bytes, int V,
                                                         const int* __restrict__ vbase,
                                                         float* __restrict__ out_verts,
                                                         uint8_t* __restrict__ out_colors) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int o = vbase[v];
  if (vbase[v + 1] == o) return;
  if (out_verts) {
#pragma unroll
    for (int d = 0; d < 3; ++d) out_verts[(size_t)o * 3 + d] = __ldg(verts + (size_t)v * 3 + d);
  }
  if (out_colors)
    for (int b = 0; b < color_bytes; ++b)
      out_colors[(size_t)o * color_bytes + b] = __ldg(colors + (size_t)v * color_bytes + b);
}

__global__ void __launch_bounds__(256) k_cull_emit_faces(const int32_t* __restrict__ faces, int Fn,
                                                         const int* __restrict__ keep,
                                                         const int* __restrict__ fbase,
                                                         const int* __restrict__ vbase,
                                                         int32_t* __restrict__ out_faces) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= Fn || !keep[f]) return;
  const int o = fbase[f];
#pragma unroll
  for (int m = 0; m < 3; ++m)
    out_faces[(size_t)o * 3 + m] = vbase[__ldg(faces + (size_t)f * 3 + m)];
}

struct Ws : Carver {
  Ws(void* base, int V, int Fn) : Carver(base), V(V), Fn(Fn) {}
  const int V, Fn;
  int *keep = take<int>(Fn + 1), *fbase = take<int>(Fn + 1);
  int *ref = take<int>(V + 1), *vbase = take<int>(V + 1);
  CubTemp scan = cub(
      [&](size_t& b) {
        return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, Fn + 1);
      },
      [&](size_t& b) {
        return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, V + 1);
      });
};

bool sizes_ok(int V, int Fn) { return V >= 0 && Fn >= 0 && V < 0x7fffffff && Fn < 0x7fffffff; }

bool params_ok(const XrdCullParams& P) { return P.H >= 1 && P.W >= 1; }

}  // namespace cull
}  // namespace xrd

using namespace xrd;
using namespace xrd::cull;

extern "C" int xrd_cull_visible(const float* verts, int n_verts, const float* w2c,
                                const float* depth, int n_frames, const XrdCullParams* params,
                                uint8_t* seen, void* stream_) {
  if (!params || (n_verts > 0 && (!verts || !seen))) return XRD_E_NULL;
  if (n_verts < 0 || n_frames < 1 || n_frames > XRD_CULL_MAX_FRAMES || !params_ok(*params))
    return XRD_E_SHAPE;
  if (!w2c || !depth) return XRD_E_NULL;
  if (n_verts == 0) return XRD_OK;
  cudaStream_t stream = (cudaStream_t)stream_;
  k_cull_visible<<<blocks(n_verts), 256, (size_t)n_frames * 12 * sizeof(float), stream>>>(
      verts, n_verts, w2c, depth, n_frames, *params, seen);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" size_t xrd_cull_workspace_bytes(int n_verts, int n_faces) {
  if (!sizes_ok(n_verts, n_faces)) return 0;
  return Ws(nullptr, n_verts, n_faces).bytes();
}

extern "C" int xrd_cull_count(const uint8_t* seen, int n_verts, const int32_t* faces, int n_faces,
                              int32_t* counts, void* workspace, size_t workspace_bytes,
                              void* stream_) {
  if (!counts || !workspace || (n_verts > 0 && !seen) || (n_faces > 0 && !faces))
    return XRD_E_NULL;
  if (!sizes_ok(n_verts, n_faces)) return XRD_E_SHAPE;
  Ws L(workspace, n_verts, n_faces);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  XRD_CUDA_TRY(cudaMemsetAsync(L.ref, 0, (size_t)(n_verts + 1) * 4, stream));
  XRD_CUDA_TRY(cudaMemsetAsync(counts, 0, 3 * sizeof(int32_t), stream));
  k_cull_faces<<<blocks((long long)n_faces + 1), 256, 0, stream>>>(seen, n_verts, faces, n_faces,
                                                                   L.keep, L.ref, counts + 2);
  XRD_LAUNCH_CHECK();
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(L.scan.ptr, L.scan.bytes, L.keep, L.fbase,
                                             n_faces + 1, stream));
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(L.scan.ptr, L.scan.bytes, L.ref, L.vbase,
                                             n_verts + 1, stream));
  return copy_totals(counts, L.vbase + n_verts, L.fbase + n_faces, stream);
}

extern "C" int xrd_cull_emit(const float* verts, const uint8_t* colors, int color_bytes,
                             int n_verts, const int32_t* faces, int n_faces, float* out_verts,
                             uint8_t* out_colors, int32_t* out_faces, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  if (!workspace) return XRD_E_NULL;
  if (!sizes_ok(n_verts, n_faces) || color_bytes < 0) return XRD_E_SHAPE;
  if ((out_verts && n_verts > 0 && !verts) || (out_faces && n_faces > 0 && !faces) ||
      (out_colors && color_bytes > 0 && n_verts > 0 && !colors))
    return XRD_E_NULL;
  const Ws L(workspace, n_verts, n_faces);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!color_bytes) out_colors = nullptr;
  if (n_verts > 0 && (out_verts || out_colors)) {
    k_cull_emit_verts<<<blocks(n_verts), 256, 0, stream>>>(verts, colors, color_bytes, n_verts,
                                                           L.vbase, out_verts, out_colors);
    XRD_LAUNCH_CHECK();
  }
  if (n_faces > 0 && out_faces) {
    k_cull_emit_faces<<<blocks(n_faces), 256, 0, stream>>>(faces, n_faces, L.keep, L.fbase,
                                                           L.vbase, out_faces);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}
