// sample_pdf (slam/model_components/utils.py:31-76) for one ray on one warp: the importance
// samples of Co-SLAM's k_importance (coslam.cu) and NICE-SLAM's k_sample_pdf (nice.cu).
//   pdf  = (w[1:-1] + 1e-5) / sum, the sum in float64 rounded once to float
//   cdf  = [0, cumsum(pdf)]: the prefix sums in float64 and each rounded to float, as
//          torch.cumsum does on float32
//   bins = .5 (z[1:] + z[:-1]); u given, the det linspace, or Philox at counters 2^63 | r N + j
//   searchsorted(cdf, u, right=True), the below / above clamps, denom < 1e-5 -> 1,
//   sample = bins[below] + t (bins[above] - bins[below])
//   z_out = sort(z ++ samples), each value written at its rank.
// V, the type of z, the bins and the samples: float (Co-SLAM) or double (NICE-SLAM).  Every
// operation on them rounds as its __f*_rn / __d*_rn intrinsic.
#pragma once
#include "common.cuh"

namespace xrd {

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

// where the uniforms of the N samples of a ray come from
struct PdfDraw {
  const float* u;      // [R][N], or NULL
  const float* lin_u;  // [N] the det linspace (u NULL, det)
  int det;
  uint64_t seed;       // u NULL, !det: Philox, counters above 2^63 (disjoint from the jitter's)
};

// pdf[0, M) and cdf[0, M] (M = S - 2) of the inner weights weight(1) .. weight(M), the bin
// midpoints bins[0, S - 1) of z[0, S), and zall[0, S) = z.  Ends with the warp in sync.
template <class V, class Weight>
__device__ __forceinline__ void pdf_cdf(const Weight& weight, const V* z, int S, float* pdf,
                                        float* cdf, V* bins, V* zall, int lane) {
  const int M = S - 2;
  double part = 0.0;
  for (int j = lane; j < M; j += 32) {
    const float w = __fadd_rn(weight(j + 1), 1e-5f);
    pdf[j] = w;
    part += (double)w;
  }
  const float sum = (float)warp_sum_d(part);
  for (int j = lane; j < S - 1; j += 32) bins[j] = mul_rn((V)0.5, add_rn(z[j + 1], z[j]));
  for (int k = lane; k < S; k += 32) zall[k] = z[k];
  __syncwarp();
  // lane owns the contiguous run [j0, j1) of the pdf; exclusive scan of the run totals
  const int C = (M + 31) / 32, j0 = min(M, lane * C), j1 = min(M, j0 + C);
  double run = 0.0;
  for (int j = j0; j < j1; ++j) {
    const float q = __fdiv_rn(pdf[j], sum);
    pdf[j] = q;
    run += (double)q;
  }
  double pre = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double v = __shfl_up_sync(0xffffffffu, pre, o);
    if (lane >= o) pre += v;
  }
  pre -= run;
  for (int j = j0; j < j1; ++j) {
    pre += (double)pdf[j];
    cdf[j + 1] = (float)pre;
  }
  if (lane == 0) cdf[0] = 0.f;
  __syncwarp();
}

// The N samples of ray r by the inverse of the cdf of pdf_cdf: into zall[S, S + N) and, if not
// NULL, z_samples[0, N) in draw order.  Ends with the warp in sync.
template <class V>
__device__ __forceinline__ void invert_cdf(const PdfDraw& d, int r, int S, int N, const float* cdf,
                                           const V* bins, V* zall, V* z_samples, int lane) {
  const int M = S - 2;
  for (int j = lane; j < N; j += 32) {
    float u;
    if (d.u) {
      u = d.u[(size_t)r * N + j];
    } else if (d.det) {
      u = d.lin_u[j];
    } else {
      float q[4];
      philox4(d.seed, (1ull << 63) | ((uint64_t)r * N + j), q);
      u = q[0];
    }
    // searchsorted(cdf, u, right=True): the first index whose cdf exceeds u, in [0, M + 1]
    int lo = 0, hi = M + 1;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (cdf[m] <= u) lo = m + 1; else hi = m;
    }
    const int below = max(lo - 1, 0), above = min(lo, M);
    const float c0 = cdf[below];
    float den = __fsub_rn(cdf[above], c0);
    if (den < 1e-5f) den = 1.f;
    const float t = __fdiv_rn(__fsub_rn(u, c0), den);
    const V b0 = bins[below];
    const V z = add_rn(b0, mul_rn((V)t, sub_rn(bins[above], b0)));
    zall[S + j] = z;
    if (z_samples) z_samples[j] = z;
  }
  __syncwarp();
}

// out[0, T) = zall[0, T) sorted: each value written at its rank, ties in index order
template <class V>
__device__ __forceinline__ void rank_merge(const V* zall, int T, V* out, int lane) {
  for (int e = lane; e < T; e += 32) {
    const V v = zall[e];
    int rank = 0;
    for (int q = 0; q < T; ++q) {
      const V x = zall[q];
      rank += (x < v) || (x == v && q < e);
    }
    out[rank] = v;
  }
}

}  // namespace xrd
