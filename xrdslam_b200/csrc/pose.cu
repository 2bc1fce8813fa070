// Camera poses on the device (SURVEY row A6; "next" row f1): axis-angle + translation ->
// c2w 4x4 and the backward, so that a whole bundle-adjustment iteration needs no host autograd.
// Restates slam/utils/opt_pose.py:77-95 (OptimizablePose.axis_angle_to_rotation_matrix):
//   theta = |w| ; theta ~ 0 -> R = I (no gradient) ; k = w / theta ; K = skew(k)
//   R = I + sin(theta) K + (1 - cos(theta)) K K
// and :51-55 matrix(): c2w = [[R, t], [0 0 0 1]].
#include "common.cuh"
#include "../../include/xrdslam_b200.h"

namespace xrd {
namespace pose {

__device__ __forceinline__ void skew(const float k[3], float K[9]) {
  K[0] = 0.f;   K[1] = -k[2]; K[2] = k[1];
  K[3] = k[2];  K[4] = 0.f;   K[5] = -k[0];
  K[6] = -k[1]; K[7] = k[0];  K[8] = 0.f;
}
__device__ __forceinline__ void mm3(const float A[9], const float B[9], float C[9]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C[i * 3 + j] = fmaf(A[i * 3 + 2], B[6 + j], fmaf(A[i * 3 + 1], B[3 + j], A[i * 3] * B[j]));
}

__global__ void k_fwd(int n, const float* rot, const float* trans, float* c2w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float w[3] = {rot[i * 3], rot[i * 3 + 1], rot[i * 3 + 2]};
  const float th = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  float R[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
  if (th > 1e-8f) {  // torch.allclose(angle, 0): |angle| <= 1e-8
    const float k[3] = {w[0] / th, w[1] / th, w[2] / th};
    float K[9], K2[9];
    skew(k, K);
    mm3(K, K, K2);
    // 1 - cos(th) as 2 sin^2(th / 2): 1.f - cosf(th) cancels to 0 for th < ~3e-4, which costs
    // the backward's (dk - (dk . k) k) / th up to ~1e3 ulp of |G| there
    const float s = sinf(th), h = sinf(0.5f * th), c1 = 2.f * h * h;
#pragma unroll
    for (int q = 0; q < 9; ++q) R[q] = (q % 4 == 0 ? 1.f : 0.f) + K[q] * s + c1 * K2[q];
  }
  float* M = c2w + (size_t)i * 16;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    M[r * 4] = R[r * 3]; M[r * 4 + 1] = R[r * 3 + 1]; M[r * 4 + 2] = R[r * 3 + 2];
    M[r * 4 + 3] = trans[i * 3 + r];
  }
  M[12] = M[13] = M[14] = 0.f; M[15] = 1.f;
}

// d loss / d (w, t) += chain of d loss / d c2w through the formula above (what autograd does):
//   R = I + s K(k) + c1 K(k)^2,  k = w / th
//   dL/dK = s G + c1 (G K^T + K^T G),  G = dL/dR ;  dL/dk from the skew layout
//   dL/dth (explicit) = cos(th) <G,K> + sin(th) <G,K^2>
//   dL/dw = (dL/dk - (dL/dk . k) k) / th + dL/dth * k
__global__ void k_bwd(int n, const float* rot, const float* d_c2w, const unsigned char* fixed,
                      float* d_rot, float* d_trans) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (fixed && fixed[i]) return;
  const float* G4 = d_c2w + (size_t)i * 16;
#pragma unroll
  for (int r = 0; r < 3; ++r) d_trans[i * 3 + r] += G4[r * 4 + 3];
  const float w[3] = {rot[i * 3], rot[i * 3 + 1], rot[i * 3 + 2]};
  const float th = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(th > 1e-8f)) return;  // identity branch: no gradient
  float G[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) G[r * 3 + c] = G4[r * 4 + c];
  const float k[3] = {w[0] / th, w[1] / th, w[2] / th};
  float K[9], K2[9], Kt[9], GKt[9], KtG[9];
  skew(k, K);
  mm3(K, K, K2);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) Kt[r * 3 + c] = K[c * 3 + r];
  mm3(G, Kt, GKt);
  mm3(Kt, G, KtG);
  const float s = sinf(th), co = cosf(th), h = sinf(0.5f * th), c1 = 2.f * h * h;  // as in k_fwd
  float dK[9], gK = 0.f, gK2 = 0.f;
#pragma unroll
  for (int q = 0; q < 9; ++q) {
    dK[q] = s * G[q] + c1 * (GKt[q] + KtG[q]);
    gK = fmaf(G[q], K[q], gK);
    gK2 = fmaf(G[q], K2[q], gK2);
  }
  // K = [[0,-k2,k1],[k2,0,-k0],[-k1,k0,0]]
  const float dk[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
  const float dth = co * gK + s * gK2;
  const float dot = dk[0] * k[0] + dk[1] * k[1] + dk[2] * k[2];
#pragma unroll
  for (int d = 0; d < 3; ++d) d_rot[i * 3 + d] += (dk[d] - dot * k[d]) / th + dth * k[d];
}

}  // namespace pose
}  // namespace xrd

using namespace xrd;

extern "C" int xrd_pose_matrices(int n_poses, const float* rot, const float* trans, float* c2w,
                                 void* stream) {
  if (n_poses <= 0) return XRD_OK;
  if (!rot || !trans || !c2w) return XRD_E_NULL;
  pose::k_fwd<<<(n_poses + 63) / 64, 64, 0, (cudaStream_t)stream>>>(n_poses, rot, trans, c2w);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_pose_matrices_grads(int n_poses, const float* rot, const float* d_c2w,
                                       const uint8_t* fixed, float* d_rot, float* d_trans,
                                       void* stream) {
  if (n_poses <= 0) return XRD_OK;
  if (!rot || !d_c2w || !d_rot || !d_trans) return XRD_E_NULL;
  pose::k_bwd<<<(n_poses + 63) / 64, 64, 0, (cudaStream_t)stream>>>(n_poses, rot, d_c2w, fixed,
                                                                      d_rot, d_trans);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
