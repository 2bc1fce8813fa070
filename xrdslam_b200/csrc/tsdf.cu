// Block-sparse TSDF fusion of RGB-D keyframes and coloured marching cubes over its blocks
// (sm_90a), plus the connected components used by clean_mesh.
//
// Replaces (reference @ f0366f20):
//   slam/common/common.py:622-663  get_mesh_from_RGBD: open3d ScalableTSDFVolume integrate of
//                                  every keyframe, then extract_triangle_mesh, on the host
//   slam/common/common.py:666-711  clean_mesh: trimesh.graph.connected_components
// Semantics (fixed here, documented in include/xrdslam_b200.h): 16^3-voxel blocks keyed by
// packed (bx, by, bz); the allocated set is the sorted union of the blocks every frame touches;
// frame k updates only the blocks it touched, each voxel owned by one thread that applies the
// frames in order; every fp32 operation is an explicit round-to-nearest intrinsic.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "mc_device.cuh"
#include "mc_table.cuh"

namespace xrd {
namespace tsdf {

constexpr int kRes = 16;                 // voxels per block edge
constexpr int kVox = kRes * kRes * kRes; // voxels per block
constexpr int kBias = 1 << 20;           // 21 signed bits per axis
constexpr unsigned long long kNone = ~0ull;

__host__ __device__ __forceinline__ unsigned long long pack(int bx, int by, int bz) {
  return ((unsigned long long)(bx + kBias) << 42) | ((unsigned long long)(by + kBias) << 21) |
         (unsigned long long)(bz + kBias);
}
__device__ __forceinline__ void unpack(unsigned long long k, int b[3]) {
  b[0] = (int)((k >> 42) & 0x1fffff) - kBias;
  b[1] = (int)((k >> 21) & 0x1fffff) - kBias;
  b[2] = (int)(k & 0x1fffff) - kBias;
}

// row r of a [3][4] rigid transform applied to (x, y, z, 1), left to right
__device__ __forceinline__ float xform(const float* T, int r, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(T + 4 * r), x),
                                       __fmul_rn(__ldg(T + 4 * r + 1), y)),
                             __fmul_rn(__ldg(T + 4 * r + 2), z)),
                   __ldg(T + 4 * r + 3));
}

__device__ __forceinline__ bool depth_ok(float d, float depth_trunc) {
  return d > 0.f && !(d > depth_trunc);
}

// ---- allocation ------------------------------------------------------------------------------
// one thread per (frame, sampled pixel): up to 8 (block key, frame) candidates, kNone if unused
__global__ void __launch_bounds__(256) k_alloc_points(const float* __restrict__ depth,
                                                       const float* __restrict__ c2w, int K,
                                                       int H, int W, int Hs, int Ws,
                                                       XrdTsdfParams P,
                                                       unsigned long long* __restrict__ key,
                                                       int* __restrict__ frame) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = (long long)Hs * Ws;
  if (t >= (long long)K * per) return;
  const int f = (int)(t / per);
  const int r = (int)(t % per);
  const int v = (r / Ws) * P.stride, u = (r % Ws) * P.stride;
  unsigned long long* out = key + t * 8;
#pragma unroll
  for (int c = 0; c < 8; ++c) { out[c] = kNone; frame[t * 8 + c] = f; }
  const float d = __ldg(depth + ((size_t)f * H + v) * W + u);
  if (!depth_ok(d, P.depth_trunc)) return;
  const float x = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, P.cx), d), P.fx);
  const float y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, P.cy), d), P.fy);
  const float* T = c2w + (size_t)f * 12;
  const float bl = __fmul_rn(P.voxel_length, (float)kRes);
  int lo[3], n[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float p = xform(T, a, x, y, d);
    const float l = floorf(__fdiv_rn(__fsub_rn(p, P.sdf_trunc), bl));
    const float h = floorf(__fdiv_rn(__fadd_rn(p, P.sdf_trunc), bl));
    if (!(l >= (float)-kBias && h < (float)(kBias - 1))) return;  // outside the key range / NaN
    lo[a] = (int)l;
    n[a] = min((int)h - lo[a], 1) + 1;
  }
  int c = 0;
  for (int dx = 0; dx < n[0]; ++dx)
    for (int dy = 0; dy < n[1]; ++dy)
      for (int dz = 0; dz < n[2]; ++dz) out[c++] = pack(lo[0] + dx, lo[1] + dy, lo[2] + dz);
}

// head[i] = 1 at the first candidate of each allocated block (sorted keys); head[n] = 0
__global__ void k_alloc_heads(const unsigned long long* __restrict__ key, long long n,
                              int* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  head[i] = i < n && key[i] != kNone && (i == 0 || key[i] != key[i - 1]);
}

__global__ void k_alloc_emit(const unsigned long long* __restrict__ key,
                             const int* __restrict__ frame, const int* __restrict__ head,
                             const int* __restrict__ rank, long long n, int words,
                             unsigned long long* __restrict__ keys, uint32_t* __restrict__ masks) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || key[i] == kNone) return;
  const int b = rank[i] + head[i] - 1;
  if (head[i]) keys[b] = key[i];
  const int f = frame[i];
  atomicOr(masks + (size_t)b * words + (f >> 5), 1u << (f & 31));
}

// ---- integration -----------------------------------------------------------------------------
// one thread per voxel; the 4096 voxels of a block share its touched-frame list, so the frame
// loop is uniform across the CUDA block.  tsdf, weight and colour stay in registers.
__global__ void __launch_bounds__(256) k_integrate(
    const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ masks, int words,
    const float* __restrict__ depth, const uint8_t* __restrict__ color,
    const float* __restrict__ w2c, int H, int W, XrdTsdfParams P, float* __restrict__ tsdf,
    float* __restrict__ weight, float* __restrict__ rgb) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long b = g / kVox;
  const int v = (int)(g % kVox);
  int bk[3];
  unpack(keys[b], bk);
  const int idx[3] = {v >> 8, (v >> 4) & 15, v & 15};
  const float bl = __fmul_rn(P.voxel_length, (float)kRes);
  float p[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    p[a] = __fadd_rn(__fmul_rn((float)bk[a], bl), __fmul_rn((float)idx[a] + 0.5f, P.voxel_length));
  float ts = tsdf[g], w = weight[g], c0 = rgb[g * 3], c1 = rgb[g * 3 + 1], c2 = rgb[g * 3 + 2];
  bool upd = false;
  const uint32_t* m = masks + b * words;
  for (int wd = 0; wd < words; ++wd) {
    uint32_t bits = __ldg(m + wd);
    while (bits) {
      const int f = wd * 32 + __ffs(bits) - 1;
      bits &= bits - 1;
      const float* T = w2c + (size_t)f * 12;
      const float z = xform(T, 2, p[0], p[1], p[2]);
      if (!(z > 0.f)) continue;
      const float x = xform(T, 0, p[0], p[1], p[2]);
      const float y = xform(T, 1, p[0], p[1], p[2]);
      const float fu = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(P.fx, x), z), P.cx), 0.5f));
      const float fv = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(P.fy, y), z), P.cy), 0.5f));
      if (!(fu >= 0.f && fu < (float)W && fv >= 0.f && fv < (float)H)) continue;
      const size_t pix = ((size_t)f * H + (int)fv) * W + (int)fu;
      const float d = __ldg(depth + pix);
      if (!depth_ok(d, P.depth_trunc)) continue;
      const float qa = __fdiv_rn(__fsub_rn(fu, P.cx), P.fx);
      const float qb = __fdiv_rn(__fsub_rn(fv, P.cy), P.fy);
      const float mult = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(qa, qa), __fmul_rn(qb, qb)), 1.f));
      const float sdf = __fmul_rn(__fsub_rn(d, z), mult);
      if (sdf <= -P.sdf_trunc) continue;
      const float t = fminf(1.f, __fdiv_rn(sdf, P.sdf_trunc));
      const float w1 = __fadd_rn(w, 1.f);
      ts = __fdiv_rn(__fadd_rn(__fmul_rn(ts, w), t), w1);
      c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, w), (float)__ldg(color + pix * 3)), w1);
      c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, w), (float)__ldg(color + pix * 3 + 1)), w1);
      c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, w), (float)__ldg(color + pix * 3 + 2)), w1);
      w = w1;
      upd = true;
    }
  }
  if (upd) {
    tsdf[g] = ts; weight[g] = w;
    rgb[g * 3] = c0; rgb[g * 3 + 1] = c1; rgb[g * 3 + 2] = c2;
  }
}

// ---- marching cubes over blocks ----------------------------------------------------------------
// The dense kernels of mesh.cu cannot be reused as they are: a cube here is used only when all
// 8 corners exist (neighbour blocks may be unallocated) and have weight > 0, and a crossed edge
// gets a vertex only if a used cube references it, so vertex ownership is decided by a marking
// pass rather than by the sign change alone.  The interpolation, the affine and the edge ->
// vertex-id lookup are the shared helpers of mc_device.cuh.

// nbr[b][c - 1] = id of the block at offset (c >> 2 & 1, c >> 1 & 1, c & 1), or -1
__global__ void k_neighbours(const unsigned long long* __restrict__ keys, int n_blocks,
                             int* __restrict__ nbr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_blocks * 7) return;
  const int b = t / 7, c = t % 7 + 1;
  int bk[3];
  unpack(keys[b], bk);
  const int o[3] = {(c >> 2) & 1, (c >> 1) & 1, c & 1};
  int id = -1;
  if (bk[0] + o[0] < kBias && bk[1] + o[1] < kBias && bk[2] + o[2] < kBias) {
    const unsigned long long q = pack(bk[0] + o[0], bk[1] + o[1], bk[2] + o[2]);
    int lo = 0, hi = n_blocks;  // lower bound
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys[mid] < q) lo = mid + 1; else hi = mid;
    }
    if (lo < n_blocks && keys[lo] == q) id = lo;
  }
  nbr[t] = id;
}

// global voxel index of local position (i, j, k) in 0..16 of block b, or -1 if its block is
// not allocated
__device__ __forceinline__ long long voxel_at(const int* __restrict__ nbr, long long b, int i,
                                              int j, int k) {
  const int c = ((i >> 4) << 2) | ((j >> 4) << 1) | (k >> 4);
  const long long nb = c ? (long long)nbr[b * 7 + c - 1] : b;
  if (nb < 0) return -1;
  return nb * kVox + ((i & 15) << 8) + ((j & 15) << 4) + (k & 15);
}

// per voxel: the case of the cube anchored there (tcnt = its triangles, 0 if the cube is not
// used); clears the owned-edge flags.  Index n: the scan sentinels.
__global__ void __launch_bounds__(256) k_classify(const float* __restrict__ tsdf,
                                                  const float* __restrict__ weight,
                                                  const int* __restrict__ nbr, long long n,
                                                  uint8_t* __restrict__ cases,
                                                  uint32_t* __restrict__ flags,
                                                  int* __restrict__ vcnt,
                                                  int* __restrict__ tcnt) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n) return;
  if (g == n) { vcnt[n] = 0; tcnt[n] = 0; return; }
  flags[g] = 0;
  const long long b = g / kVox;
  const int v = (int)(g % kVox);
  const int i = v >> 8, j = (v >> 4) & 15, k = v & 15;
  int cs = 0;
  bool used = true;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const long long q = voxel_at(nbr, b, i + ((c >> 2) & 1), j + ((c >> 1) & 1), k + (c & 1));
    if (q < 0 || !(__ldg(weight + q) > 0.f)) { used = false; break; }
    cs |= (int)(__ldg(tsdf + q) < 0.f) << c;
  }
  cases[g] = (uint8_t)cs;
  tcnt[g] = used ? (int)c_mc_ntri[cs] : 0;
}

// every used cube marks the edges its triangles reference on the edge's owner voxel
__global__ void __launch_bounds__(256) k_mark(const int* __restrict__ nbr, long long n,
                                              const uint8_t* __restrict__ cases,
                                              const int* __restrict__ tcnt,
                                              uint32_t* __restrict__ flags) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const int nt = tcnt[g];
  if (!nt) return;
  const int cs = cases[g];
  int emask = 0;
  for (int e = 0; e < 3 * nt; ++e) emask |= 1 << c_mc_tri[cs][e];
  const long long b = g / kVox;
  const int v = (int)(g % kVox);
  const int i = v >> 8, j = (v >> 4) & 15, k = v & 15;
  for (int e = 0; e < 12; ++e) {
    if (!((emask >> e) & 1)) continue;
    const long long q = voxel_at(nbr, b, i + c_mc_edge_off[e][0], j + c_mc_edge_off[e][1],
                                 k + c_mc_edge_off[e][2]);
    atomicOr(flags + q, 1u << c_mc_edge_axis[e]);
  }
}

__global__ void k_vcount(const uint32_t* __restrict__ flags, long long n, int* __restrict__ vcnt) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) vcnt[g] = __popc(flags[g]);
}

__global__ void __launch_bounds__(256) k_verts(const unsigned long long* __restrict__ keys,
                                               const float* __restrict__ tsdf,
                                               const float* __restrict__ rgb,
                                               const int* __restrict__ nbr, long long n,
                                               float voxel_length,
                                               const uint32_t* __restrict__ flags,
                                               const int* __restrict__ vbase,
                                               float* __restrict__ verts,
                                               float* __restrict__ colors) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const int fl = flags[g];
  if (!fl) return;
  const long long b = g / kVox;
  const int v = (int)(g % kVox);
  const int idx[3] = {v >> 8, (v >> 4) & 15, v & 15};
  int bk[3];
  unpack(keys[b], bk);
  const float bl = __fmul_rn(voxel_length, (float)kRes);
  const float half = __fmul_rn(voxel_length, 0.5f);
  float o[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = __fmul_rn((float)bk[d], bl);
  const float v0 = __ldg(tsdf + g);
  int id = vbase[g];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!((fl >> a) & 1)) continue;
    const long long q = voxel_at(nbr, b, idx[0] + (a == 0), idx[1] + (a == 1), idx[2] + (a == 2));
    const float t = mc::edge_t(0.f, v0, __ldg(tsdf + q));
    float c[3] = {(float)idx[0], (float)idx[1], (float)idx[2]};
    c[a] = __fadd_rn(c[a], t);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      verts[(size_t)id * 3 + d] = mc::world(c[d], voxel_length, half, 1.f, o[d]);
      const float k0 = __ldg(rgb + g * 3 + d), k1 = __ldg(rgb + q * 3 + d);
      colors[(size_t)id * 3 + d] = __fdiv_rn(__fadd_rn(k0, __fmul_rn(t, __fsub_rn(k1, k0))), 255.f);
    }
    ++id;
  }
}

__global__ void __launch_bounds__(256) k_faces(const int* __restrict__ nbr, long long n,
                                               const uint8_t* __restrict__ cases,
                                               const int* __restrict__ tcnt,
                                               const uint32_t* __restrict__ flags,
                                               const int* __restrict__ vbase,
                                               const int* __restrict__ tbase,
                                               int* __restrict__ faces) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const int nt = tcnt[g];
  if (!nt) return;
  const int cs = cases[g];
  const long long b = g / kVox;
  const int v = (int)(g % kVox);
  const int i = v >> 8, j = (v >> 4) & 15, k = v & 15;
  const int f0 = tbase[g];
  for (int t = 0; t < nt; ++t) {
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      const int e = c_mc_tri[cs][3 * t + m];
      const long long q = voxel_at(nbr, b, i + c_mc_edge_off[e][0], j + c_mc_edge_off[e][1],
                                   k + c_mc_edge_off[e][2]);
      faces[(size_t)(f0 + t) * 3 + m] = mc::edge_vertex(vbase[q], flags[q], c_mc_edge_axis[e]);
    }
  }
}

// ---- connected components ----------------------------------------------------------------------
// Union-find: a root is only ever hooked (CAS) below a smaller root, so parent[x] <= x always and
// every component ends at its minimum vertex id whatever the scheduling.
__device__ __forceinline__ int cc_root(volatile int* parent, int x) {
  int y;
  while ((y = parent[x]) != x) x = y;
  return x;
}

__global__ void k_cc_init(int* parent, int V) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V) parent[i] = i;
}

__global__ void k_cc_hook(const int* __restrict__ faces, long long n_edges, int* parent) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const long long f = e / 3;
  const int m = (int)(e % 3);
  int a = faces[f * 3 + m], b = faces[f * 3 + (m + 1) % 3];
  while (true) {
    a = cc_root(parent, a);
    b = cc_root(parent, b);
    if (a == b) return;
    if (a > b) { const int s = a; a = b; b = s; }
    if (atomicCAS(parent + b, b, a) == b) return;
  }
}

__global__ void k_cc_compress(int* parent, int V) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V) parent[i] = cc_root(parent, i);
}

// ---- workspaces ---------------------------------------------------------------------------------
struct AllocWs : Carver {
  AllocWs(void* base, int K, int H, int W, int stride)
      : Carver(base), n((long long)K * ((H + stride - 1) / stride) * ((W + stride - 1) / stride) * 8) {}
  const long long n;  // candidates
  unsigned long long *key_in = take<unsigned long long>(n), *key_out = take<unsigned long long>(n);
  int *frame_in = take<int>(n), *frame_out = take<int>(n);
  int *head = take<int>(n + 1), *rank = take<int>(n + 1);
  CubTemp temp = cub(
      [&](size_t& b) {
        return cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned long long*)nullptr,
                                               (unsigned long long*)nullptr, (const int*)nullptr,
                                               (int*)nullptr, (int)n);
      },
      [&](size_t& b) {
        return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr,
                                             (int)(n + 1));
      });
};

bool alloc_shape_ok(int K, int H, int W, int stride) {
  if (K < 1 || H < 1 || W < 1 || stride < 1) return false;
  const long long Hs = (H + stride - 1) / stride, Ws = (W + stride - 1) / stride;
  return (long long)K * Hs * Ws * 8 < 0x7fffffffLL;  // CUB's int item count holds n + 1
}

bool params_ok(const XrdTsdfParams& P) {
  // at most two blocks per axis around a point: 2 * sdf_trunc below one block edge
  return P.voxel_length > 0.f && P.sdf_trunc > 0.f && P.fx > 0.f && P.fy > 0.f &&
         P.stride >= 1 && 2.f * P.sdf_trunc < P.voxel_length * (float)kRes;
}

struct McWs : Carver {
  McWs(void* base, int n_blocks) : Carver(base), n_blocks(n_blocks) {}
  const int n_blocks;
  const long long n = (long long)n_blocks * kVox;  // voxels
  int* nbr = take<int>((size_t)n_blocks * 7);
  uint8_t* cases = take<uint8_t>(n);
  uint32_t* flags = take<uint32_t>(n);
  int *vcnt = take<int>(n + 1), *tcnt = take<int>(n + 1);
  int *vbase = take<int>(n + 1), *tbase = take<int>(n + 1);
  CubTemp scan = cub([&](size_t& b) {
    return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, (int)(n + 1));
  });
};

bool blocks_ok(int n_blocks) {
  return n_blocks >= 1 && (long long)n_blocks * kVox < 0x7fffffffLL;
}

}  // namespace tsdf
}  // namespace xrd

using namespace xrd;
using namespace xrd::tsdf;

extern "C" size_t xrd_tsdf_alloc_workspace_bytes(int K, int H, int W, int stride) {
  if (!alloc_shape_ok(K, H, W, stride)) return 0;
  return AllocWs(nullptr, K, H, W, stride).bytes();
}

extern "C" int xrd_tsdf_alloc_count(const float* depth, const float* c2w, int K, int H, int W,
                                    const XrdTsdfParams* params, int32_t* n_blocks,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
  if (!depth || !c2w || !params || !n_blocks || !workspace) return XRD_E_NULL;
  const XrdTsdfParams P = *params;
  if (!params_ok(P) || !alloc_shape_ok(K, H, W, P.stride)) return XRD_E_SHAPE;
  AllocWs L(workspace, K, H, W, P.stride);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int Hs = (H + P.stride - 1) / P.stride, Ws = (W + P.stride - 1) / P.stride;
  k_alloc_points<<<blocks(L.n / 8), 256, 0, stream>>>(depth, c2w, K, H, W, Hs, Ws, P, L.key_in,
                                                      L.frame_in);
  XRD_LAUNCH_CHECK();
  XRD_CUDA_TRY(cub::DeviceRadixSort::SortPairs(L.temp.ptr, L.temp.bytes, L.key_in, L.key_out,
                                               L.frame_in, L.frame_out, (int)L.n, 0, 64, stream));
  k_alloc_heads<<<blocks(L.n + 1), 256, 0, stream>>>(L.key_out, L.n, L.head);
  XRD_LAUNCH_CHECK();
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(L.temp.ptr, L.temp.bytes, L.head, L.rank,
                                             (int)(L.n + 1), stream));
  return copy_totals(n_blocks, L.rank + L.n, nullptr, stream);
}

extern "C" int xrd_tsdf_alloc_emit(int K, int H, int W, const XrdTsdfParams* params,
                                   int n_blocks, int64_t* keys, uint32_t* masks, void* workspace,
                                   size_t workspace_bytes, void* stream_) {
  if (!params || !keys || !masks || !workspace) return XRD_E_NULL;
  const XrdTsdfParams P = *params;
  if (!params_ok(P) || !alloc_shape_ok(K, H, W, P.stride) || n_blocks < 1) return XRD_E_SHAPE;
  const AllocWs L(workspace, K, H, W, P.stride);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int words = (K + 31) / 32;
  XRD_CUDA_TRY(cudaMemsetAsync(masks, 0, (size_t)n_blocks * words * 4, stream));
  k_alloc_emit<<<blocks(L.n), 256, 0, stream>>>(L.key_out, L.frame_out, L.head, L.rank, L.n,
                                                words, reinterpret_cast<unsigned long long*>(keys),
                                                masks);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_tsdf_integrate(const int64_t* keys, const uint32_t* masks, int n_blocks,
                                  const float* depth, const uint8_t* color, const float* w2c,
                                  int K, int H, int W, const XrdTsdfParams* params, float* tsdf,
                                  float* weight, float* color_acc, void* stream_) {
  if (!keys || !masks || !depth || !color || !w2c || !params || !tsdf || !weight || !color_acc)
    return XRD_E_NULL;
  const XrdTsdfParams P = *params;
  if (!params_ok(P) || !blocks_ok(n_blocks) || K < 1 || H < 1 || W < 1) return XRD_E_SHAPE;
  cudaStream_t stream = (cudaStream_t)stream_;
  const long long n = (long long)n_blocks * kVox;
  k_integrate<<<blocks(n), 256, 0, stream>>>(reinterpret_cast<const unsigned long long*>(keys),
                                             masks, (K + 31) / 32, depth, color, w2c, H, W, P,
                                             tsdf, weight, color_acc);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" size_t xrd_tsdf_mc_workspace_bytes(int n_blocks) {
  if (!blocks_ok(n_blocks)) return 0;
  return McWs(nullptr, n_blocks).bytes();
}

extern "C" int xrd_tsdf_mc_count(const int64_t* keys, int n_blocks, const float* tsdf,
                                 const float* weight, int32_t* counts, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  if (!keys || !tsdf || !weight || !counts || !workspace) return XRD_E_NULL;
  if (!blocks_ok(n_blocks)) return XRD_E_SHAPE;
  McWs L(workspace, n_blocks);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const long long n = L.n;
  const auto* k = reinterpret_cast<const unsigned long long*>(keys);
  k_neighbours<<<blocks((long long)n_blocks * 7), 256, 0, stream>>>(k, n_blocks, L.nbr);
  XRD_LAUNCH_CHECK();
  k_classify<<<blocks(n + 1), 256, 0, stream>>>(tsdf, weight, L.nbr, n, L.cases, L.flags, L.vcnt,
                                                L.tcnt);
  XRD_LAUNCH_CHECK();
  k_mark<<<blocks(n), 256, 0, stream>>>(L.nbr, n, L.cases, L.tcnt, L.flags);
  XRD_LAUNCH_CHECK();
  k_vcount<<<blocks(n), 256, 0, stream>>>(L.flags, n, L.vcnt);
  XRD_LAUNCH_CHECK();
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(L.scan.ptr, L.scan.bytes, L.vcnt, L.vbase,
                                             (int)(n + 1), stream));
  XRD_CUDA_TRY(cub::DeviceScan::ExclusiveSum(L.scan.ptr, L.scan.bytes, L.tcnt, L.tbase,
                                             (int)(n + 1), stream));
  return copy_totals(counts, L.vbase + n, L.tbase + n, stream);
}

extern "C" int xrd_tsdf_mc_emit(const int64_t* keys, int n_blocks, const float* tsdf,
                                const float* color_acc, const XrdTsdfParams* params,
                                float* verts, float* colors, int32_t* faces, void* workspace,
                                size_t workspace_bytes, void* stream_) {
  if (!keys || !tsdf || !color_acc || !params || !workspace) return XRD_E_NULL;
  if (!blocks_ok(n_blocks) || !params_ok(*params)) return XRD_E_SHAPE;
  const McWs L(workspace, n_blocks);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  const long long n = L.n;
  if (verts && colors) {
    k_verts<<<blocks(n), 256, 0, stream>>>(reinterpret_cast<const unsigned long long*>(keys), tsdf,
                                           color_acc, L.nbr, n, params->voxel_length, L.flags,
                                           L.vbase, verts, colors);
    XRD_LAUNCH_CHECK();
  }
  if (faces) {
    k_faces<<<blocks(n), 256, 0, stream>>>(L.nbr, n, L.cases, L.tcnt, L.flags, L.vbase, L.tbase,
                                           faces);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}

extern "C" int xrd_tsdf_components(const int32_t* faces, int n_faces, int n_verts,
                                   int32_t* labels, void* stream_) {
  if (!labels || (n_faces > 0 && !faces)) return XRD_E_NULL;
  if (n_faces < 0 || n_verts < 0) return XRD_E_SHAPE;
  if (n_verts == 0) return XRD_OK;
  cudaStream_t stream = (cudaStream_t)stream_;
  k_cc_init<<<blocks(n_verts), 256, 0, stream>>>(labels, n_verts);
  XRD_LAUNCH_CHECK();
  if (n_faces > 0) {
    const long long ne = (long long)n_faces * 3;
    k_cc_hook<<<blocks(ne), 256, 0, stream>>>(faces, ne, labels);
    XRD_LAUNCH_CHECK();
  }
  k_cc_compress<<<blocks(n_verts), 256, 0, stream>>>(labels, n_verts);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
