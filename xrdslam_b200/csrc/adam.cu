// Multi-tensor Adam step in ONE launch (SURVEY row B3: `Optimizers.optimizer_step_all`,
// slam/engine/optimizers.py:125-162 -> torch.optim.Adam.step; the update rule restated from
// torch/optim/adam.py `_single_tensor_adam`, amsgrad=False, maximize=False):
//   g  = grad (+ weight_decay * p)
//   m += (g - m) * (1 - beta1)                  (Tensor.lerp_)
//   v  = v * beta2 + (1 - beta2) * g * g        (mul_ + addcmul_)
//   p -= (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// HBM-bound: 4 reads + 3 writes per element (1.64 M hash floats -> 46 MB, ~8 us at 6.5 TB/s);
// float4 accesses, one (tensor, chunk) pair per block.  zero_grad folds `zero_grad_all` into
// the same pass (the gradient is overwritten with zeros after it is read).
#include "common.cuh"
#include "../../include/xrdslam_b200.h"

namespace xrd {
namespace adam {

struct Args {
  XrdAdamTensor t[XRD_ADAM_MAX_TENSORS];
  int n;
  int zero_grad;
};

__device__ __forceinline__ void upd(float& p, float& g, float& m, float& v, const XrdAdamTensor& T,
                                    float step_size, float inv_sqrt_bc2) {
  float gg = g;
  if (T.weight_decay != 0.f) gg = __fadd_rn(gg, __fmul_rn(T.weight_decay, p));
  m = __fadd_rn(m, __fmul_rn(__fsub_rn(gg, m), 1.0f - T.beta1));
  v = __fadd_rn(__fmul_rn(v, T.beta2), __fmul_rn(__fmul_rn(1.0f - T.beta2, gg), gg));
  const float denom = __fadd_rn(__fmul_rn(sqrtf(v), inv_sqrt_bc2), T.eps);
  p = __fsub_rn(p, __fmul_rn(step_size, __fdiv_rn(m, denom)));
}

__global__ void __launch_bounds__(256) k_adam(const Args A) {
  const XrdAdamTensor& T = A.t[blockIdx.y];
  const float lr = T.dyn ? T.dyn[0] : T.lr;
  const float step_size = lr / (T.dyn ? T.dyn[1] : T.bias_correction1);
  const float inv_sqrt_bc2 = 1.0f / sqrtf(T.dyn ? T.dyn[2] : T.bias_correction2);
  const long long n = T.n;
  const bool vec = ((((uintptr_t)T.param | (uintptr_t)T.grad | (uintptr_t)T.exp_avg |
                      (uintptr_t)T.exp_avg_sq) & 15) == 0);
  const bool masked = T.row_mask != nullptr;
  const long long n4 = (vec && (!masked || (T.row_len & 3) == 0)) ? n / 4 : 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    if (masked && !T.row_mask[(i * 4) / T.row_len]) {  // row_len % 4 == 0: one row per float4
      // a kept row holds its parameter and moments, but zero_grad still clears its gradient
      if (A.zero_grad) reinterpret_cast<float4*>(T.grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    float4 p = reinterpret_cast<float4*>(T.param)[i];
    float4 g = reinterpret_cast<float4*>(T.grad)[i];
    float4 m = reinterpret_cast<float4*>(T.exp_avg)[i];
    float4 v = reinterpret_cast<float4*>(T.exp_avg_sq)[i];
    upd(p.x, g.x, m.x, v.x, T, step_size, inv_sqrt_bc2);
    upd(p.y, g.y, m.y, v.y, T, step_size, inv_sqrt_bc2);
    upd(p.z, g.z, m.z, v.z, T, step_size, inv_sqrt_bc2);
    upd(p.w, g.w, m.w, v.w, T, step_size, inv_sqrt_bc2);
    reinterpret_cast<float4*>(T.param)[i] = p;
    reinterpret_cast<float4*>(T.exp_avg)[i] = m;
    reinterpret_cast<float4*>(T.exp_avg_sq)[i] = v;
    if (A.zero_grad) reinterpret_cast<float4*>(T.grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    if (masked && !T.row_mask[i / T.row_len]) {
      if (A.zero_grad) T.grad[i] = 0.f;
      continue;
    }
    float p = T.param[i], g = T.grad[i], m = T.exp_avg[i], v = T.exp_avg_sq[i];
    upd(p, g, m, v, T, step_size, inv_sqrt_bc2);
    T.param[i] = p; T.exp_avg[i] = m; T.exp_avg_sq[i] = v;
    if (A.zero_grad) T.grad[i] = 0.f;
  }
}

}  // namespace adam
}  // namespace xrd

using namespace xrd;

extern "C" int xrd_adam_step(const XrdAdamTensor* tensors, int n_tensors, int zero_grad,
                             void* stream) {
  if (n_tensors <= 0) return XRD_OK;
  if (!tensors) return XRD_E_NULL;
  for (int base = 0; base < n_tensors; base += XRD_ADAM_MAX_TENSORS) {
    adam::Args A;
    A.n = n_tensors - base < XRD_ADAM_MAX_TENSORS ? n_tensors - base : XRD_ADAM_MAX_TENSORS;
    A.zero_grad = zero_grad;
    long long nmax = 0;
    for (int i = 0; i < A.n; ++i) {
      A.t[i] = tensors[base + i];
      if (!A.t[i].param || !A.t[i].grad || !A.t[i].exp_avg || !A.t[i].exp_avg_sq) return XRD_E_NULL;
      if (A.t[i].n < 0 || (!A.t[i].dyn && (A.t[i].bias_correction1 <= 0.f || A.t[i].bias_correction2 <= 0.f)))
        return XRD_E_SHAPE;
      if (A.t[i].row_mask && A.t[i].row_len < 1) return XRD_E_SHAPE;
      if (A.t[i].n > nmax) nmax = A.t[i].n;
    }
    long long bx = (nmax / 4 + 255) / 256;
    if (bx < 1) bx = 1;
    if (bx > num_sms() * 8) bx = num_sms() * 8;
    adam::k_adam<<<dim3((unsigned)bx, (unsigned)A.n), 256, 0, (cudaStream_t)stream>>>(A);
    XRD_LAUNCH_CHECK();
  }
  return XRD_OK;
}
