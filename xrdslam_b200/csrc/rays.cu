// Shared front-end on the device (SURVEY rows A2 / A7, "next" row f1):
//   world-frame rays from camera-frame directions and a per-ray pose row
//     rays_d = sum_j dir_cam[j] * c2w[id][:3, j],   rays_o = c2w[id][:3, 3]
//   (slam/common/common.py:39-53 get_rays_from_uv; slam/algorithms/coslam.py:208-216 per-ray
//   pose gather `poses_all[ids_all]`), and the reduction of d loss / d rays into d loss / d c2w
//   that torch does with an index_put(accumulate) sort + scatter -- here one launch with
//   shared-memory accumulators.
#include "common.cuh"
#include "../../include/xrdslam_b200.h"

namespace xrd {
namespace rays {

constexpr int MAXP = 64;  // poses accumulated in shared memory (bundle window is ~5-20)

struct P {
  int R, n_poses;
  const float* dirs; const int64_t* ids; const float* poses;
  float *rays_o, *rays_d;
  const float *d_rays_o, *d_rays_d;
  float* d_poses;
};

// Row of the pose table a ray reads, or -1 when the id is out of range.  torch raises an
// IndexError for `poses_all[ids_all]` there (coslam.py:208-216); an asynchronous kernel cannot,
// so an out-of-range ray gets NaN rays (the loss turns NaN: loud) and contributes no gradient
// -- never an out-of-bounds access.
__device__ __forceinline__ int pose_row(const P& p, int r) {
  long long id = p.ids ? p.ids[r] : 0;
  if (id < 0) id += p.n_poses;  // python indexing: -1 = the current frame, appended last
  return (id < 0 || id >= p.n_poses) ? -1 : (int)id;
}

__global__ void __launch_bounds__(256) k_fwd(const P p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.R) return;
  const int row = pose_row(p, r);
  if (row < 0) {
    const float nan = __int_as_float(0x7fc00000);
#pragma unroll
    for (int c = 0; c < 3; ++c) p.rays_d[r * 3 + c] = p.rays_o[r * 3 + c] = nan;
    return;
  }
  const float* M = p.poses + (size_t)row * 16;
  const float d0 = p.dirs[r * 3], d1 = p.dirs[r * 3 + 1], d2 = p.dirs[r * 3 + 2];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.rays_d[r * 3 + c] = __fadd_rn(__fadd_rn(__fmul_rn(d0, M[c * 4]), __fmul_rn(d1, M[c * 4 + 1])),
                                    __fmul_rn(d2, M[c * 4 + 2]));
    p.rays_o[r * 3 + c] = M[c * 4 + 3];
  }
}

__global__ void __launch_bounds__(256) k_bwd(const P p) {
  __shared__ float acc[MAXP * 12];
  const bool use_smem = p.n_poses <= MAXP;
  if (use_smem) {
    for (int i = threadIdx.x; i < p.n_poses * 12; i += blockDim.x) acc[i] = 0.f;
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  // whole warps iterate together (r0 is warp-uniform) so the shuffles below are convergent
  for (int r0 = (blockIdx.x * blockDim.x + threadIdx.x) - lane; r0 < p.R; r0 += gridDim.x * blockDim.x) {
    const int r = r0 + lane;
    const int id = (r < p.R) ? pose_row(p, r) : -1;
    const bool live = id >= 0;  // out-of-range ids contribute nothing
    float v[12];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float gd = (live && p.d_rays_d) ? p.d_rays_d[r * 3 + c] : 0.f;
      const float go = (live && p.d_rays_o) ? p.d_rays_o[r * 3 + c] : 0.f;
#pragma unroll
      for (int j = 0; j < 3; ++j) v[c * 4 + j] = live ? gd * p.dirs[r * 3 + j] : 0.f;
      v[c * 4 + 3] = go;
    }
    // rays of one frame are contiguous: usually the whole warp shares the pose row ->
    // shuffle-reduce and issue 12 atomics per warp instead of 12 per lane
    const int id0 = __shfl_sync(0xffffffffu, id, 0);
    const bool uniform = __all_sync(0xffffffffu, id == id0 || !live) && id0 >= 0;
    if (uniform) {
#pragma unroll
      for (int k = 0; k < 12; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
      }
      if (lane == 0) {
        float* a = use_smem ? acc + id0 * 12 : nullptr;
#pragma unroll
        for (int k = 0; k < 12; ++k) {
          if (use_smem) atomicAdd(a + k, v[k]);
          else atomicAdd(p.d_poses + (size_t)id0 * 16 + k, v[k]);
        }
      }
    } else if (live) {
#pragma unroll
      for (int k = 0; k < 12; ++k) {
        if (use_smem) atomicAdd(acc + id * 12 + k, v[k]);
        else atomicAdd(p.d_poses + (size_t)id * 16 + k, v[k]);
      }
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < p.n_poses * 12; i += blockDim.x)
      if (acc[i] != 0.f) atomicAdd(p.d_poses + (size_t)(i / 12) * 16 + (i % 12), acc[i]);
  }
}

// ---- pixel sampling for a window of frames (SURVEY rows A1 / A3 / A8-A10) -------------------
constexpr int MAXF = 32;
struct PixP {
  XrdPixelSampleCfg c;
  const float* depth[MAXF];
  const float* rgb[MAXF];
  const int64_t* indices;
  float *dirs, *o_depth, *o_rgb;
  int64_t *pose_ids, *ij;
};

__global__ void __launch_bounds__(256) k_pixels(const PixP p) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = p.c.n_per_frame;
  if (q >= p.c.n_frames * n) return;
  const int f = q / n;
  const int w = p.c.W1 - p.c.W0;
  const long long idx = p.indices[q];
  const int ii = (int)(idx % w) + p.c.W0;       // column
  const int jj = (int)(idx / w) + p.c.H0;       // row
  const size_t pix = (size_t)jj * p.c.W + ii;
  p.o_depth[q] = p.depth[f][pix];
  const float* c = p.rgb[f] + pix * 3;
  p.o_rgb[q * 3] = c[0]; p.o_rgb[q * 3 + 1] = c[1]; p.o_rgb[q * 3 + 2] = c[2];
  // dirs = [(i - cx) / fx, -(j - cy) / fy, -1]   (common.py:45-47)
  p.dirs[q * 3] = __fdiv_rn(__fsub_rn((float)ii, p.c.cx), p.c.fx);
  p.dirs[q * 3 + 1] = -__fdiv_rn(__fsub_rn((float)jj, p.c.cy), p.c.fy);
  p.dirs[q * 3 + 2] = -1.0f;
  p.pose_ids[q] = f;
  if (p.ij) { p.ij[q * 2] = ii; p.ij[q * 2 + 1] = jj; }
}

}  // namespace rays
}  // namespace xrd

using namespace xrd;

extern "C" int xrd_sample_pixels(const XrdPixelSampleCfg* cfg, const float* const* depth_imgs,
                                 const float* const* rgb_imgs, const int64_t* indices, float* dirs,
                                 float* depth, float* rgb, int64_t* pose_ids, int64_t* ij,
                                 void* stream) {
  if (!cfg || !depth_imgs || !rgb_imgs || !indices || !dirs || !depth || !rgb || !pose_ids)
    return XRD_E_NULL;
  if (cfg->n_frames < 1 || cfg->n_frames > rays::MAXF || cfg->n_per_frame < 0) return XRD_E_SHAPE;
  if (cfg->H0 < 0 || cfg->W0 < 0 || cfg->H1 > cfg->H || cfg->W1 > cfg->W || cfg->H1 <= cfg->H0 ||
      cfg->W1 <= cfg->W0)
    return XRD_E_SHAPE;
  const int total = cfg->n_frames * cfg->n_per_frame;
  if (total == 0) return XRD_OK;
  rays::PixP p{};
  p.c = *cfg;
  for (int f = 0; f < cfg->n_frames; ++f) {
    if (!depth_imgs[f] || !rgb_imgs[f]) return XRD_E_NULL;
    p.depth[f] = depth_imgs[f]; p.rgb[f] = rgb_imgs[f];
  }
  p.indices = indices; p.dirs = dirs; p.o_depth = depth; p.o_rgb = rgb; p.pose_ids = pose_ids;
  p.ij = ij;
  rays::k_pixels<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_rays_from_poses(int n_rays, const float* dirs_cam, const int64_t* pose_ids,
                                   const float* poses, int n_poses, float* rays_o, float* rays_d,
                                   void* stream) {
  if (n_rays <= 0) return XRD_OK;
  if (!dirs_cam || !poses || !rays_o || !rays_d) return XRD_E_NULL;
  if (n_poses < 1) return XRD_E_SHAPE;
  rays::P p{};
  p.R = n_rays; p.n_poses = n_poses; p.dirs = dirs_cam; p.ids = pose_ids; p.poses = poses;
  p.rays_o = rays_o; p.rays_d = rays_d;
  rays::k_fwd<<<(n_rays + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_rays_pose_grads(int n_rays, const float* dirs_cam, const int64_t* pose_ids,
                                   int n_poses, const float* d_rays_o, const float* d_rays_d,
                                   float* d_poses, void* stream) {
  if (!d_poses) return XRD_E_NULL;
  if (n_poses < 1) return XRD_E_SHAPE;
  XRD_CUDA_TRY(cudaMemsetAsync(d_poses, 0, (size_t)n_poses * 16 * sizeof(float), (cudaStream_t)stream));
  if (n_rays <= 0) return XRD_OK;
  if (!dirs_cam || (!d_rays_o && !d_rays_d)) return XRD_E_NULL;
  rays::P p{};
  p.R = n_rays; p.n_poses = n_poses; p.dirs = dirs_cam; p.ids = pose_ids;
  p.d_rays_o = d_rays_o; p.d_rays_d = d_rays_d; p.d_poses = d_poses;
  int blocks = (n_rays + 255) / 256;
  if (blocks > num_sms()) blocks = num_sms();
  rays::k_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(p);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
