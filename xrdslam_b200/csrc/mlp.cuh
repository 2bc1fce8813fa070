// Wide per-point MLP layers on [feature][point] activations (points contiguous): the GEMM
// (Vox-Fusion decoder, Point-SLAM colour decoder) and the weight-gradient reduction (NICE-SLAM,
// Vox-Fusion, Point-SLAM).  Kernels and launchers are in mlp.cu; both run under the calling
// thread's xrd_debug_gemm_mode.
#pragma once
#include "common.cuh"

namespace xrd {

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_SOFTPLUS100 = 2, ACT_SIGMOID = 3 };

//   C[m][n] = epi( sum_k A(m,k) * B[k][n] ),   A(m,k) = transA ? A[k*lda+m] : A[m*lda+k]
//   epi(v)  = act(v + bias[m]);  zeroed where relu_mask[m][n] <= 0 (optional: backward of a
//             relu layer);  act_out[m][n] = epi(v) (optional);  + addend[m][n] (optional);
//             accumulate: C += that.
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

// out[j*sj + i*si] += sum_p Brow_j[p] (masked) * Arow_i[p];  bias[j] += sum_p Brow_j[p] (masked)
struct DwJob {
  const float* A; int nA;          // rows of Pp floats
  const float* B; int nB;
  const uint32_t* mask;            // per-point relu mask word (bit j) or NULL
  float* out; int sj, si;
  float* bias;                     // or NULL
};
constexpr int DW_MAX_JOBS = 32;
struct DwParams {
  DwJob jobs[DW_MAX_JOBS];
  int n_jobs, P, Pp, chunk;
};

cudaError_t launch_gemm(const GemmArgs& G, cudaStream_t stream);
// sets Q.chunk (points per CTA) on the fp32 SIMT path
cudaError_t launch_dw(DwParams& Q, cudaStream_t stream);

}  // namespace xrd
