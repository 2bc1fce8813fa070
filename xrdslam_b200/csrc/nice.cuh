// Parameters and launcher of the NICE-SLAM decoder kernels (nice.cu), which Point-SLAM also runs
// on its kNN-interpolated features.
#pragma once
#include "common.cuh"

namespace xrd {
namespace nice {

struct Grid {
  const float* data = nullptr;
  float* grad = nullptr;
  int nx = 1, ny = 1, nz = 1;
};

struct DecParams {
  int P, S;
  const double* z = nullptr;
  const float *rays_o, *rays_d;
  double bmin[3] = {0.0, 0.0, 0.0}, bmax[3] = {1.0, 1.0, 1.0};
  Grid ga;          // own grid
  Grid gb;          // fine decoder: the middle grid (no gradient); data == NULL otherwise
  XrdNiceDecoder dec = {};
  // outputs / inputs per point (SoA)
  float* out[4] = {};        // fwd: out[k][p] (n_out rows)
  const float* dout[4] = {}; // bwd: d loss / d out[k][p]
  uint32_t* masks = nullptr; // [5][P]
  float* acts = nullptr;     // trainable: rows of Pp floats: e[93] h0..h4[160] c[c_dim] | bwd: dh[160] gm[93] pf[3]
  int Pp = 0;
  float* dp = nullptr;       // [3][P] d loss / d point, accumulated across the decoder passes
  int need_dp = 0;
  // Point-SLAM reuses this decoder with a kNN-interpolated feature instead of a grid:
  const float* zf = nullptr;     // float32 sample depths (z == NULL)
  const float* ext_c = nullptr;  // [c_dim][P] feature rows (ga.data == NULL)
  float* ext_dc = nullptr;       // [c_dim][P] gradient w.r.t. the feature rows
  float embed_scale = 1.0f;      // 1 (NICE: sin(p B)) or 2*pi (Point-SLAM: sin(2 pi p B))
};

// k_decoder_fwd (bwd false) or k_decoder_bwd over the D.P points: sizes the shared memory for
// D.dec.c_dim and runs one CTA per tile of points, at most one per SM
cudaError_t launch_decoder(const DecParams& D, bool bwd, cudaStream_t stream);

}  // namespace nice
}  // namespace xrd
