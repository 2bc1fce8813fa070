// Co-SLAM render-and-optimise step, fused forward + backward (sm_90a).
//
// Replaces (reference @ f0366f20): slam/models/joint_encoding.py:250-344
// render_rays, :483-507 run_network, :463-481 query_color_sdf (tcnn HashGrid +
// OneBlob, slam/model_components/encodings_coslam.py:39-75; decoders
// slam/model_components/decoder_coslam.py:139-163), :346-406 sdf2weights /
// raw2outputs, :94-147 get_loss_dict (+ slam/model_components/utils.py:100-186)
// and the autograd backward of the whole chain.
//
// Kernels
//   k_sample   one warp per ray: merge the 32 uniform + 11 depth-guided samples,
//              stratified jitter, batch-global counts n_fs / n_sdf / n_valid.
//   k_fused    persistent CTAs over tiles of NR rays (NR*S points, one thread per
//              point for the gathers).  Per-point fp32 record in shared memory, dense:
//                [feat32 | blob48 | geo15 | sdf | h1_32 | c1_32 | raw4]   (stride 164)
//              The decoder runs on the tensor cores: every warp pushes its own 32
//              points through mma.sync m16n8k8 TF32 tiles whose A fragments are read
//              straight from the records (stride 164 = 4 mod 32 -> conflict-free) and
//              whose B fragments are the transposed weights staged in shared memory;
//              3xTF32 error compensation keeps fp32-level parity (cfg.precision).
//              forward -> per-ray composite + loss gradient (one warp per ray) ->
//              layer-by-layer backward that overwrites activations with their
//              gradients in place; weight gradients are 16x8 MMA tiles with the
//              points on the K axis, accumulated in registers for the whole launch;
//              the hash backward runs in the MMA fragment layout (lane (g,t) owns
//              level 4*nt+t of rows g, g+8) and scatters corner pairs: one red.global.add.v4.f32
//              for two x-adjacent corners in one 16-byte chunk of d_table, red.v2 otherwise.
//   k_fused_g  the same arithmetic through the same device functions, scheduled as
//              independent groups of warps with named barriers, one m-tile per warp, a
//              132-float record with OneBlob in compact form and a balanced
//              point-parallel hash backward (see its comment).
//   k_fused_c  the tile kernel for a separate colour hash grid (Co-SLAM oneGrid=False,
//              decoder_coslam.py:113-136 ColorSDFNet): a second 16-level gather into the record,
//              the 95-input colour decoder, and the colour grid's hash backward (scatter into
//              d_table_c, d loss / d xn).
//   k_finalize loss accumulators -> the 4 weighted loss terms.
//   k_importance  hierarchical sampling between a coarse and a fine pass (training_n_importance
//              > 0): the coarse weights, sample_pdf, the sorted merge and the fine pass's counts.
#include <math.h>

#include "common.cuh"
#include "sample_pdf.cuh"

namespace xrd {
namespace coslam {

constexpr int kL = XRD_MAX_LEVELS;
constexpr int kBins = 16;
// Per-point records (floats); stride == 4 (mod 32) keeps 128-bit LDS conflict-free.
// Dense (tile kernel, k_query): [feat32 | blob48 | geo15 | sdf | h1 32 | c1 32 | raw4], stride 164.
constexpr int R_FEAT = 0, R_BLOB = 32, R_GEO = 80, R_SDF = 95, R_H1 = 96, R_C1 = 128,
              R_RAW = 160, REC = 164;
// Compact (grouped kernel), stride 132: the 48 OneBlob bins are kept in compact form
// (blob_compact_dim), so that the decoder-input columns outside the OneBlob block sit at their
// own index: [feat 0..31 | blob] for the SDF decoder, [blob | geo 48..62 | sdf 63] for the colour
// decoder.  The tile kernel keeps the dense record: on the compact one its gradient pass is
// slower (DESIGN.md section 4.1).
constexpr int G_FEAT = 0, G_BLOB = 32, G_GEO = 48, G_SDF = 63, G_H1 = 64, G_C1 = 96, G_RAW = 128,
              GREC = 132;
// Colour grid (k_fused_c, k_query_c), stride 196: the colour grid's features sit between OneBlob
// and geo, so that the 95 colour-decoder inputs [blob48 | cfeat32 | geo15] and the zero-weight
// sdf column are one contiguous block of 12 k-steps:
//   [feat32 | blob48 | cfeat32 | geo15 | sdf | h1 32 | c1 32 | raw4]
constexpr int C_CFEAT = 80, C_GEO = 112, C_SDF = 127, C_H1 = 128, C_C1 = 160, C_RAW = 192,
              CREC = 196;
// Colour grid, forward only (CGF), stride 132: h1 overwrites the hash features once the first
// GEMM has read them, and c1 overwrites h1 once the second has; nothing needs them afterwards.
// [feat32 -> h1 -> c1 | blob48 | cfeat32 | geo15 | sdf | raw4].  This is what lets a render
// pass without depth (256 samples: one ray of 256 points per tile) fit in shared memory.
constexpr int F_H = 0, F_RAW = 128, FREC = 132;
// per-layout offsets for the code the kernels share (CG: colour-grid record, CGF: its
// forward-only form)
template <bool COMPACT, bool CG = false, bool CGF = false>
struct Rec {
  static constexpr int N = COMPACT ? GREC : CGF ? FREC : CG ? CREC : REC,
                       GEO = COMPACT ? G_GEO : CG ? C_GEO : R_GEO,
                       SDF = COMPACT ? G_SDF : CG ? C_SDF : R_SDF,
                       H1 = COMPACT ? G_H1 : CGF ? F_H : CG ? C_H1 : R_H1,
                       C1 = COMPACT ? G_C1 : CGF ? F_H : CG ? C_C1 : R_C1,
                       RAW = COMPACT ? G_RAW : CGF ? F_RAW : CG ? C_RAW : R_RAW;
};
struct GridDev {
  float scale[kL];
  uint32_t res[kL], size[kL], offset[kL], hashed[kL];
  uint32_t magic[kL];  // floor(2^32 / size): q = umulhi(index, magic) <= index/size, off by <= 1
  int n_levels;
  double bmin[3], binv[3];  // 1/(max-min): gradients only; the forward divides (index parity)
  double bmax[3];
};

struct Params {
  // rays
  int R, S, Rg;  // Rg: rays of the global (all-rank) batch the loss means run over
  const float *rays_o, *rays_d, *target_s, *target_d;
  const float* z_vals;  // [R,S] (written by k_sample)
  // grid + mlp
  GridDev g;
  const float* table;
  const float *w_sdf0, *w_sdf1, *w_col0, *w_col1;
  // cfg
  float trunc, depth_trunc, w_rgb, w_depth, w_sdf, w_fs;
  float ls[4];
  // outputs
  float *rgb, *depth, *disp, *acc, *depth_var, *raw;
  // grads
  float *d_table, *d_w_sdf0, *d_w_sdf1, *d_w_col0, *d_w_col1, *d_rays_o, *d_rays_d;
  // workspace
  const int* counts;  // n_fs, n_sdf, n_valid
  double* loss_acc;   // 4 sums
  int NR;             // rays per tile
  int n_tiles;
};
// k_fused_c: the colour grid on top (normalised coordinates come from g's bound)
struct ParamsC : Params {
  GridDev gc;
  const float* table_c;
  float* d_table_c;
};

// ------------------------------------------------------------------ sample ---
struct SampleParams {
  int R, S, n_a, n_b, perturb, has_depth;
  const float *target_d, *lin_uniform, *lin_range, *lin_nodepth, *lin_full, *noise;
  float trunc, depth_trunc;
  uint64_t seed;
  const uint64_t* seed_dev;
  float* z_vals;
  int* counts;
};

// The loss normalisers' counts (SURVEY Q9) of one sample at depth zv on a ray of target depth d:
// free-space samples (c_fs) and samples inside the truncation band (c_sdf).
__device__ __forceinline__ void count_sample(float zv, float d, float trunc, int& c_fs, int& c_sdf) {
  const bool front = zv < __fsub_rn(d, trunc);
  const bool back = zv > __fadd_rn(d, trunc);
  c_fs += front;
  c_sdf += (!front && !back && d > 0.f);
}
// One warp's counts into counts[0..2] = n_fs, n_sdf, n_valid (c_valid: lane 0's).
__device__ __forceinline__ void add_counts(int* counts, int c_fs, int c_sdf, int c_valid, int lane) {
  c_fs = warp_sum_i(c_fs);
  c_sdf = warp_sum_i(c_sdf);
  if (lane == 0) {
    if (c_fs) atomicAdd(&counts[0], c_fs);
    if (c_sdf) atomicAdd(&counts[1], c_sdf);
    if (c_valid) atomicAdd(&counts[2], c_valid);
  }
}

__global__ void __launch_bounds__(128) k_sample(SampleParams p) {
  __shared__ float zs[4][260];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + warp;
  int c_fs = 0, c_sdf = 0, c_valid = 0;
  if (r < p.R) {
    float* z = zs[warp];
    const int S = p.S;
    float d = 0.f;
    if (p.has_depth) {
      d = p.target_d[r];
      const bool nodepth = d <= 0.f;  // z_samples[target_d <= 0] = linspace(near, far)
      // rank-merge of the two sorted lists (values equal torch.sort's output)
      for (int k = lane; k < S; k += 32) {
        float v;
        int rank;
        if (k < p.n_a) {
          v = p.lin_uniform[k];
          int c = 0;
          for (int j = 0; j < p.n_b; ++j) {
            float b = nodepth ? p.lin_nodepth[j] : __fadd_rn(p.lin_range[j], d);
            c += (b < v);
          }
          rank = k + c;
        } else {
          int j = k - p.n_a;
          v = nodepth ? p.lin_nodepth[j] : __fadd_rn(p.lin_range[j], d);
          int c = 0;
          for (int i = 0; i < p.n_a; ++i) c += (p.lin_uniform[i] <= v);
          rank = j + c;
        }
        z[rank] = v;
      }
    } else {
      for (int k = lane; k < S; k += 32) z[k] = p.lin_full[k];
    }
    __syncwarp();
    for (int k = lane; k < S; k += 32) {
      float zv = z[k];
      if (p.perturb) {
        float lo = (k == 0) ? zv : __fmul_rn(0.5f, __fadd_rn(zv, z[k - 1]));
        float hi = (k == S - 1) ? zv : __fmul_rn(0.5f, __fadd_rn(z[k + 1], zv));
        float u;
        if (p.noise) {
          u = p.noise[(size_t)r * S + k];
        } else {
          float q[4];
          philox4(p.seed_dev ? *p.seed_dev : p.seed, (uint64_t)r * S + k, q);
          u = q[0];
        }
        zv = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), u));
      }
      p.z_vals[(size_t)r * S + k] = zv;
      if (p.has_depth) count_sample(zv, d, p.trunc, c_fs, c_sdf);
    }
    if (p.has_depth && lane == 0) c_valid = (d > 0.f && d < p.depth_trunc);
  }
  if (p.has_depth) add_counts(p.counts, c_fs, c_sdf, c_valid, lane);
}

// --------------------------------------------------------------- encoding ---

// Per-level constants, staged in SHARED memory: the level index differs between the lanes
// of a warp in the hash backward (fragment layout: l = 4 nt + t) and in k_encode, and a
// lane-varying index into the kernel-parameter constant bank serialises
// (ncu source view: ~20 % of the samples of k_fused sat on these loads).
struct __align__(16) Lv {
  float scale;
  uint32_t res, size, offset;
  uint32_t hashed, magic, pad0, pad1;
};

__device__ __forceinline__ void load_levels(Lv* s, const GridDev& g) {
  if (threadIdx.x < kL) {
    const int l = threadIdx.x;
    Lv v;
    v.scale = g.scale[l]; v.res = g.res[l]; v.size = g.size[l]; v.offset = g.offset[l];
    v.hashed = g.hashed[l]; v.magic = g.magic[l]; v.pad0 = v.pad1 = 0;
    s[l] = v;
  }
}

__device__ __forceinline__ uint32_t grid_index(const Lv& L, uint32_t x, uint32_t y, uint32_t z) {
  const uint32_t size = L.size;
  uint32_t index;
  if (L.hashed) {
    index = x ^ (y * 2654435761u) ^ (z * 805459861u);
  } else {
    // dense stride walk (stride <= size is true for all three dims on a dense level)
    const uint32_t res = L.res;
    index = x + y * res + z * res * res;
  }
  // index % size: sizes of hashed levels are powers of two; in-range dense cells are < size
  if ((size & (size - 1)) == 0) {
    index &= size - 1;
  } else if (index >= size) {  // points outside the bound wrap around (tcnn does not clamp)
    index -= __umulhi(index, L.magic) * size;  // exact remainder or remainder + size
    if (index >= size) index -= size;
    if (index >= size) index -= size;
  }
  return index + L.offset;
}

// The 8 trilinear corners of cell c on level L: corner k is (c + (k & 1), c + (k >> 1 & 1),
// c + (k >> 2)).
__device__ __forceinline__ void corner_indices(const Lv& L, const uint32_t c[3], uint32_t idx[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    idx[k] = grid_index(L, c[0] + (k & 1), c[1] + ((k >> 1) & 1), c[2] + ((k >> 2) & 1));
}

// Corner pairs.  Corners k and k + 1 (k even) differ only in x.  On a hashed level x + 1 = x ^ 1
// for even x, so the two are entries 2j and 2j + 1; on a dense level they are idx and idx + 1.
// Level offsets are even (level sizes are multiples of 8 entries), so in both cases, and for the
// wrap of out-of-box points on dense levels, the rule is: the pair is one 16-byte chunk of the
// table iff i1 == (i0 ^ 1).  That holds for about half of all pairs.
// d_table[i0] += g0, d_table[i1] += g1: one red.global.add.v4 for a pair in one chunk, two
// red.global.add.v2 otherwise, as mutually exclusive predicated instructions (no divergent branch
// per pair).  `d_table` must be 16-byte aligned (the launchers check it).  The gathers stay 8-byte
// loads: paired 16-byte loads measured no faster in the forward and slower in the hash backward
// (DESIGN.md section 4.1).
__device__ __forceinline__ void scatter_corner_pair(float* __restrict__ d_table, uint32_t i0,
                                                    uint32_t i1, float2 g0, float2 g1) {
  const bool swap = i0 & 1u;  // in a chunk, i0 is the upper half when it is odd
  const float2 lo = swap ? g1 : g0, hi = swap ? g0 : g1;
  asm volatile(
      "{\n\t.reg .pred pp;\n\t.reg .b32 t, e;\n\t.reg .u64 a0, a1;\n\t"
      "xor.b32 t, %0, 1;\n\t"
      "setp.eq.u32 pp, t, %1;\n\t"
      "and.b32 e, %0, -2;\n\t"
      "selp.b32 e, e, %0, pp;\n\t"
      "mad.wide.u32 a0, e, 8, %2;\n\t"
      "mad.wide.u32 a1, %1, 8, %2;\n\t"
      "@pp red.global.add.v4.f32 [a0], {%3, %4, %5, %6};\n\t"
      "@!pp red.global.add.v2.f32 [a0], {%7, %8};\n\t"
      "@!pp red.global.add.v2.f32 [a1], {%9, %10};\n\t}"
      ::"r"(i0), "r"(i1), "l"(d_table), "f"(lo.x), "f"(lo.y), "f"(hi.x), "f"(hi.y), "f"(g0.x),
      "f"(g0.y), "f"(g1.x), "f"(g1.y)
      : "memory");
}

// d_table[idx[k]] += wk (g0, g1) over the 8 corners, wk the trilinear weight of corner k for the
// cell fractions w (rounded as in level_feature).
__device__ __forceinline__ void scatter_corners(float* __restrict__ d_table, const uint32_t idx[8],
                                                const float w[3], float g0, float g1) {
#pragma unroll
  for (int k = 0; k < 8; k += 2) {
    const float wy = (k & 2) ? w[1] : 1.f - w[1], wz = (k & 4) ? w[2] : 1.f - w[2];
    const float wa = (1.f - w[0]) * wy * wz, wb = w[0] * wy * wz;  // corners k, k + 1
    scatter_corner_pair(d_table, idx[k], idx[k + 1], make_float2(wa * g0, wa * g1),
                        make_float2(wb * g0, wb * g1));
  }
}

__device__ __forceinline__ void pos_fract(float x, float scale, float& w, uint32_t& c) {
  float pos = fmaf(scale, x, 0.5f);
  float fl = floorf(pos);
  c = (uint32_t)(int)fl;
  w = pos - fl;
}

// normalised coordinate exactly as the reference: f32 pts -> f64 (p-min)/(max-min) -> f32
__device__ __forceinline__ float normalise(float p, double bmin, double bmax) {
  return (float)(((double)p - bmin) / (bmax - bmin));
}

// normalised coordinate of the sample at depth z on ray r: pts = o + d z in f32, as the reference
__device__ __forceinline__ void sample_xn(const Params& P, int r, float z, float xn[3]) {
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float pt = __fadd_rn(P.rays_o[r * 3 + d], __fmul_rn(P.rays_d[r * 3 + d], z));
    xn[d] = normalise(pt, P.g.bmin[d], P.g.bmax[d]);
  }
}

// quartic kernel cdf / pdf in bin units t (|t| <= 1 inside the kernel support)
__device__ __forceinline__ float qcdf(float t) {
  float t2 = t * t;
  float v = 0.9375f * t * (1.f - (2.f / 3.f) * t2 + 0.2f * t2 * t2) + 0.5f;
  return fminf(fmaxf(v, 0.f), 1.f);
}
__device__ __forceinline__ float qpdf(float t) {
  float q = 1.f - t * t;
  return (fabsf(t) < 1.f) ? 0.9375f * q * q : 0.f;
}

// OneBlob, sparse form.  out[b] = sum_{s in -1,0,1} K(e_{b+1}-x+s) - K(e_b-x+s); for image s
// only bins b0-1, b0, b0+1 (b0 = floor(16 (x-s))) are non-zero:
//   cdf(-f), cdf(1-f)-cdf(-f), 1-cdf(1-f)   with f = 16 (x-s) - b0.
__device__ __forceinline__ void blob_forward(const float xn[3], float* __restrict__ rec) {
#pragma unroll
  for (int q = 0; q < 12; ++q)
    *reinterpret_cast<float4*>(rec + R_BLOB + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int s = -1; s <= 1; ++s) {
      const float u = (xn[d] - (float)s) * (float)kBins;
      const float fl = floorf(u);
      if (fl < -1.f || fl > (float)kBins) continue;
      const int b0 = (int)fl;
      const float f = u - fl;
      const float c0 = qcdf(-f), c1 = qcdf(1.f - f);
      float* o = rec + R_BLOB + d * kBins;
      if (b0 - 1 >= 0 && b0 - 1 < kBins) o[b0 - 1] += c0;
      if (b0 >= 0 && b0 < kBins) o[b0] += c1 - c0;
      if (b0 + 1 >= 0 && b0 + 1 < kBins) o[b0 + 1] += 1.f - c1;
    }
  }
}

// Compact form of one coordinate: the three images fill windows of 3 bins that lie 15..17 bins
// apart (16 up to the rounding of x - s), so no bin gets two contributions, at most 4 of the 16
// bins are non-zero (for any x, inside the bounding box or not) and two non-zero bins never agree
// mod 4.  Bin b is kept in slot b & 3: v[b & 3] holds exactly the float of the dense sum
// (0 + contribution) and byte b & 3 of q holds b >> 2.
// Dense bin b = (q[b & 3] == b >> 2) ? v[b & 3] : 0; empty slots hold value 0.
// Per point: [v dim0 (4) | v dim1 (4) | v dim2 (4) | q dim0 | q dim1 | q dim2 | unused].
__device__ __forceinline__ void blob_compact_dim(float x, float* __restrict__ v,
                                                 uint8_t* __restrict__ q) {
  *reinterpret_cast<float4*>(v) = make_float4(0.f, 0.f, 0.f, 0.f);
  *reinterpret_cast<uint32_t*>(q) = 0u;
#pragma unroll
  for (int s = -1; s <= 1; ++s) {
    const float u = (x - (float)s) * (float)kBins;
    const float fl = floorf(u);
    if (fl < -1.f || fl > (float)kBins) continue;
    const int b0 = (int)fl;
    const float f = u - fl;
    const float c0 = qcdf(-f), c1 = qcdf(1.f - f);
    if (b0 - 1 >= 0 && b0 - 1 < kBins) { v[(b0 - 1) & 3] = 0.f + c0; q[(b0 - 1) & 3] = (uint8_t)((b0 - 1) >> 2); }
    if (b0 >= 0 && b0 < kBins) { v[b0 & 3] = 0.f + (c1 - c0); q[b0 & 3] = (uint8_t)(b0 >> 2); }
    if (b0 + 1 >= 0 && b0 + 1 < kBins) { v[(b0 + 1) & 3] = 0.f + (1.f - c1); q[(b0 + 1) & 3] = (uint8_t)((b0 + 1) >> 2); }
  }
}

// d/dx of dimension d's 16 OneBlob outputs, contracted with dblob (read through the functor)
template <typename F>
__device__ __forceinline__ float blob_backward_dim(float x, int d, F dblob) {
  float acc = 0.f;
#pragma unroll
  for (int s = -1; s <= 1; ++s) {
    const float u = (x - (float)s) * (float)kBins;
    const float fl = floorf(u);
    if (fl < -1.f || fl > (float)kBins) continue;
    const int b0 = (int)fl;
    const float f = u - fl;
    const float p0 = qpdf(-f), p1 = qpdf(1.f - f);  // d cdf(-f)/dx = -16 p0, d cdf(1-f)/dx = -16 p1
    if (b0 - 1 >= 0 && b0 - 1 < kBins) acc -= dblob(d * kBins + b0 - 1) * p0;
    if (b0 >= 0 && b0 < kBins) acc += dblob(d * kBins + b0) * (p0 - p1);
    if (b0 + 1 >= 0 && b0 + 1 < kBins) acc += dblob(d * kBins + b0 + 1) * p1;
  }
  return acc * (float)kBins;
}

// dx[d] += sum_b dblob[d*16+b] * d out_b / dx
template <typename F>
__device__ __forceinline__ void blob_backward(const float xn[3], F dblob, float dx[3]) {
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    // (fmaf(acc, 16, dx) as one rounding: keeps the v4 kernel's bits)
    float acc = blob_backward_dim(xn[d], d, dblob) * (1.0f / (float)kBins);
    dx[d] = fmaf(acc, (float)kBins, dx[d]);
  }
}

// the two features of level L at xn, trilinear over the 8 corners (all 8 loads issued first)
__device__ __forceinline__ float2 level_feature(const float* __restrict__ table, const Lv& L,
                                                const float xn[3]) {
  float w[3];
  uint32_t c[3];
  pos_fract(xn[0], L.scale, w[0], c[0]);
  pos_fract(xn[1], L.scale, w[1], c[1]);
  pos_fract(xn[2], L.scale, w[2], c[2]);
  const float2* __restrict__ tab = reinterpret_cast<const float2*>(table);
  float2 v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k)
    v[k] = __ldg(&tab[grid_index(L, c[0] + (k & 1), c[1] + ((k >> 1) & 1), c[2] + ((k >> 2) & 1))]);
  float f0 = 0.f, f1 = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float wk = ((k & 1) ? w[0] : 1.f - w[0]) * ((k & 2) ? w[1] : 1.f - w[1]) *
                     ((k & 4) ? w[2] : 1.f - w[2]);
    f0 = fmaf(wk, v[k].x, f0);
    f1 = fmaf(wk, v[k].y, f1);
  }
  return make_float2(f0, f1);
}

// Hash features of xn into a record (FEAT = 0 in both layouts): levels l0, l0 + LSTRIDE, ...
// Tile kernel and k_query: one thread per point, (l0, LSTRIDE) = (0, 1); grouped kernel: two
// threads per point, (half, 2).
template <int LSTRIDE>
__device__ __forceinline__ void encode(const float* __restrict__ table, int n_levels,
                                       const Lv* __restrict__ lv, const float xn[3],
                                       float* __restrict__ rec, int l0) {
#pragma unroll(4 / LSTRIDE)
  for (int i = 0; i < kL / LSTRIDE; ++i) {
    const int l = l0 + LSTRIDE * i;
    *reinterpret_cast<float2*>(rec + G_FEAT + 2 * l) =
        (l < n_levels) ? level_feature(table, lv[l], xn) : make_float2(0.f, 0.f);
  }
}

// NL (point, level) items of the hash backward per call (scatter (g0,g1), optional d/dx).
// Deliberately not inlined: instruction-cache footprint matters for this kernel.  It takes the
// two table pointers by value: a `const Params&` argument of a non-inlined function forces the
// caller to copy the whole ~730-byte kernel-parameter block to local memory.
// NL (point, level) items per call: the 8 NL corner loads of all levels are issued before any
// is consumed (the kernel runs at 7 warps/SM, so memory-level parallelism has to come from
// within the thread), then the 8 NL scatters.  on[h]: item present (level exists and its
// gradient is non-zero).  Levels are l0 + lstride h (tile kernel: lane t owns levels 4 nt + t).
// The items travel by value as well: an array passed by reference would live in local memory.
template <int NL>
struct LevelItems {
  float g[NL][2];  // d loss / d (f0, f1) of level l0 + lstride h
  bool on[NL];
};
template <int NL>
__device__ __noinline__ float3 hash_backward_multi(const float* __restrict__ table,
                                                   float* __restrict__ d_table,
                                                   const Lv* __restrict__ lv, int l0,
                                                   const LevelItems<NL> it, float x0, float x1,
                                                   float x2, bool need_dx, bool scatter,
                                                   int lstride = 4) {
  const float2* __restrict__ tab = reinterpret_cast<const float2*>(table);
  const auto& on = it.on;
  const auto& g = it.g;
  const float x[3] = {x0, x1, x2};
  float w[NL][3], sc[NL];
  uint32_t idx[NL][8];
#pragma unroll
  for (int h = 0; h < NL; ++h) {
    const Lv L = lv[on[h] ? l0 + lstride * h : 0];
    sc[h] = L.scale;
    uint32_t c[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) pos_fract(x[d], sc[h], w[h][d], c[d]);
    corner_indices(L, c, idx[h]);
  }
  float dx[3] = {0.f, 0.f, 0.f};
  if (need_dx) {
    float t[NL][8];
#pragma unroll
    for (int h = 0; h < NL; ++h)
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float2 v = on[h] ? __ldg(&tab[idx[h][k]]) : make_float2(0.f, 0.f);
        t[h][k] = v.x * g[h][0] + v.y * g[h][1];
      }
#pragma unroll
    for (int h = 0; h < NL; ++h) {
      const float w0 = w[h][0], w1 = w[h][1], w2 = w[h][2];
      const float* tt = t[h];
      const float d0 = (1 - w1) * (1 - w2) * (tt[1] - tt[0]) + w1 * (1 - w2) * (tt[3] - tt[2]) +
                       (1 - w1) * w2 * (tt[5] - tt[4]) + w1 * w2 * (tt[7] - tt[6]);
      const float d1 = (1 - w0) * (1 - w2) * (tt[2] - tt[0]) + w0 * (1 - w2) * (tt[3] - tt[1]) +
                       (1 - w0) * w2 * (tt[6] - tt[4]) + w0 * w2 * (tt[7] - tt[5]);
      const float d2 = (1 - w0) * (1 - w1) * (tt[4] - tt[0]) + w0 * (1 - w1) * (tt[5] - tt[1]) +
                       (1 - w0) * w1 * (tt[6] - tt[2]) + w0 * w1 * (tt[7] - tt[3]);
      if (on[h]) {
        dx[0] = fmaf(sc[h], d0, dx[0]);
        dx[1] = fmaf(sc[h], d1, dx[1]);
        dx[2] = fmaf(sc[h], d2, dx[2]);
      }
    }
  }
  if (scatter) {
#pragma unroll
    for (int h = 0; h < NL; ++h) {
      if (on[h]) scatter_corners(d_table, idx[h], w[h], g[h][0], g[h][1]);
    }
  }
  return make_float3(dx[0], dx[1], dx[2]);
}

// ------------------------------------------------------- tensor-core GEMMs ---
// mma.sync m16n8k8 tf32 (fp32 accumulate).  PREC3 = 3xTF32 error-compensated split:
// x = big + small, d += a_s*b_b + a_b*b_s + a_b*b_b  -> fp32-level accuracy.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4],
                                         const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// Operand preparation.  The tensor core reads only the upper 19 bits of a .tf32 register, so
// plain TF32 mode feeds the fp32 bits unchanged (truncation, |err| <= 2^-10 rel).  In 3xTF32
// mode big = x with the low 13 mantissa bits cleared (exactly what the hardware would see) and
// small = x - big (exact in fp32); small's own truncation error is second order (2^-20).
template <bool PREC3>
struct FragA {
  uint32_t big[4], small[4];
  __device__ __forceinline__ void set(const float (&v)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (PREC3) {
        big[i] = __float_as_uint(v[i]) & 0xffffe000u;
        small[i] = __float_as_uint(v[i] - __uint_as_float(big[i]));
      } else {
        big[i] = __float_as_uint(v[i]);
      }
    }
  }
};
template <bool PREC3>
struct FragB {
  uint32_t big[2], small[2];
  __device__ __forceinline__ void set(float v0, float v1) {
    if (PREC3) {
      big[0] = __float_as_uint(v0) & 0xffffe000u;
      big[1] = __float_as_uint(v1) & 0xffffe000u;
      small[0] = __float_as_uint(v0 - __uint_as_float(big[0]));
      small[1] = __float_as_uint(v1 - __uint_as_float(big[1]));
    } else {
      big[0] = __float_as_uint(v0);
      big[1] = __float_as_uint(v1);
    }
  }
};
template <bool PREC3>
__device__ __forceinline__ void mma(float (&d)[4], const FragA<PREC3>& a, const FragB<PREC3>& b) {
  if (PREC3) {
    mma_tf32(d, a.small, b.big);
    mma_tf32(d, a.big, b.small);
  }
  mma_tf32(d, a.big, b.big);
}

// A fragment of k-step kb of the dense 48-column OneBlob block for rows g, g + 8 of 16 compact
// records: lane t needs bins t, t + 4 of dimension kb >> 1, half kb & 1, i.e. slot t with
// quarters 2 (kb & 1) and 2 (kb & 1) + 1.
__device__ __forceinline__ void blob_frag(const float* __restrict__ mrec, int kb, int g, int t,
                                          float (&v)[4]) {
  const int d = kb >> 1;
  const uint32_t m = 2u * (uint32_t)(kb & 1);
  const float* r0 = mrec + g * GREC + G_BLOB;
  const float* r8 = r0 + 8 * GREC;
  const float a0 = r0[4 * d + t], a8 = r8[4 * d + t];
  const uint32_t q0 = reinterpret_cast<const uint8_t*>(r0 + 12 + d)[t];
  const uint32_t q8 = reinterpret_cast<const uint8_t*>(r8 + 12 + d)[t];
  v[0] = (q0 == m) ? a0 : 0.f;
  v[1] = (q8 == m) ? a8 : 0.f;
  v[2] = (q0 == m + 1) ? a0 : 0.f;
  v[3] = (q8 == m + 1) ? a8 : 0.f;
}

// C[mt][nt] += A * B for MT m-tiles of 16 records of stride STRIDE from wrec (tile kernel: 2 per
// warp, every B fragment serves both; grouped kernel: 1).
//   A[row][k] = wrec[row*STRIDE + aoff + k], except k-steps [BK0, BK0 + 6): the 48-column OneBlob
//               block, expanded from compact records
//   B[k][n]   = TRANS ? w[(noff+n)*ld + koff + k] : w[(koff+k)*ld + noff + n]
template <int KS, int NT, bool TRANS, bool PREC3, int STRIDE, int BK0 = -1, int MT>
__device__ __forceinline__ void warp_gemm(const float* __restrict__ wrec, int aoff,
                                          const float* __restrict__ w, int ld, int koff,
                                          int noff, float (&c)[MT][NT][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll 1
  for (int ks = 0; ks < KS; ++ks) {
    FragA<PREC3> a[MT];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float v[4];
      if (BK0 >= 0 && ks >= BK0 && ks < BK0 + 6) {
        blob_frag(wrec + mt * 16 * GREC, ks - BK0, g, t, v);
      } else {
        const float* r0 = wrec + (mt * 16 + g) * STRIDE + aoff + ks * 8 + t;
        v[0] = r0[0]; v[1] = r0[8 * STRIDE]; v[2] = r0[4]; v[3] = r0[8 * STRIDE + 4];
      }
      a[mt].set(v);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      FragB<PREC3> b;
      const int k0 = koff + ks * 8 + t, n0 = noff + nt * 8 + g;
      if (TRANS) b.set(w[n0 * ld + k0], w[n0 * ld + k0 + 4]);
      else b.set(w[k0 * ld + n0], w[(k0 + 4) * ld + n0]);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) mma<PREC3>(c[mt][nt], a[mt], b);
    }
  }
}

template <int MT, int NT>
__device__ __forceinline__ void zero_c(float (&c)[MT][NT][4]) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) c[mt][nt][i] = 0.f;
}

// store C (16 MT rows x 8 NT cols) into the records at column offset coff (float2 per row pair).
// RELU: max(c, 0); MASK: c where the value it replaces is > 0, else 0 (ReLU backward in place)
enum Store { PLAIN, RELU, MASK };
template <Store OP, int STRIDE, int MT, int NT>
__device__ __forceinline__ void store_c(float* __restrict__ wrec, int coff,
                                        const float (&c)[MT][NT][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      float v0 = c[mt][nt][0], v1 = c[mt][nt][1], v2 = c[mt][nt][2], v3 = c[mt][nt][3];
      float* r0 = wrec + (mt * 16 + g) * STRIDE + coff + nt * 8 + 2 * t;
      if (OP == RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
      if (OP == MASK) {
        const float2 h0 = *reinterpret_cast<float2*>(r0), h8 = *reinterpret_cast<float2*>(r0 + 8 * STRIDE);
        v0 = h0.x > 0.f ? v0 : 0.f; v1 = h0.y > 0.f ? v1 : 0.f;
        v2 = h8.x > 0.f ? v2 : 0.f; v3 = h8.y > 0.f ? v3 : 0.f;
      }
      *reinterpret_cast<float2*>(r0) = make_float2(v0, v1);
      *reinterpret_cast<float2*>(r0 + 8 * STRIDE) = make_float2(v2, v3);
    }
}

// weights in shared memory: [in][out] with padded row strides (conflict-free B fragments)
constexpr int LD0 = 40, LD1 = 24, LDC0 = 40, LDC1 = 8;
constexpr int SW0 = 0;                     // [80][40]  w_sdf0^T
constexpr int SW1 = SW0 + 80 * LD0;        // [32][24]  w_sdf1^T, cols = (geo0..14, sdf)
constexpr int SWC0 = SW1 + 32 * LD1;       // [64][40]  w_col0^T, row 63 = 0
constexpr int SWC1 = SWC0 + 64 * LDC0;     // [32][8]   w_col1^T, cols 3..7 = 0
constexpr int SW_TOTAL = SWC1 + 32 * LDC1; // 6784 floats

// weight-gradient tiles (16 in-features x 8 out-units each), global order
//   [0,2) d w_col1   [2,18) d w_col0   [18,22) d w_sdf1   [22,42) d w_sdf0
constexpr int DW_TILES = 42;

// Decoder shapes that differ with a colour grid: w_col0 has NC = 95 inputs instead of 63 (KC
// k-steps of the colour GEMM, its transpose [96][40] with row 95 = 0 in shared memory), so
// w_col1 and the end of the weight area move, and d w_col0 takes 24 weight-gradient tiles:
//   [0,2) d w_col1   [2,26) d w_col0   [26,30) d w_sdf1   [30,50) d w_sdf0
template <bool CG>
struct Wts {
  static constexpr int NC = CG ? 95 : 63, KC = CG ? 12 : 8, SWC1 = SWC0 + 8 * KC * LDC0,
                       TOTAL = SWC1 + 32 * LDC1, COL0_TILES = CG ? 24 : 16,
                       SDF1_LO = 2 + COL0_TILES, SDF0_LO = SDF1_LO + 4, DW = SDF0_LO + 20;
};
static_assert(Wts<false>::SWC1 == SWC1 && Wts<false>::TOTAL == SW_TOTAL &&
              Wts<false>::DW == DW_TILES, "one-grid decoder layout");

// A fragment values of the dense OneBlob bins (g, g + 8) of dimension bd for points p0 (k-slot t)
// and p1 (k-slot t + 4), expanded from the compact form: both bins live in slot g & 3, with
// quarters g >> 2 and (g >> 2) + 2.
__device__ __forceinline__ void blob_dw_frag(const float* __restrict__ p0,
                                             const float* __restrict__ p1, int bd, int g,
                                             float (&va)[4]) {
  const int e = g & 3;
  const uint32_t m = (uint32_t)(g >> 2);
  const float a0 = p0[G_BLOB + 4 * bd + e], a1 = p1[G_BLOB + 4 * bd + e];
  const uint32_t q0 = reinterpret_cast<const uint8_t*>(p0 + G_BLOB + 12 + bd)[e];
  const uint32_t q1 = reinterpret_cast<const uint8_t*>(p1 + G_BLOB + 12 + bd)[e];
  va[0] = (q0 == m) ? a0 : 0.f;
  va[1] = (q0 == m + 2) ? a0 : 0.f;
  va[2] = (q1 == m) ? a1 : 0.f;
  va[3] = (q1 == m + 2) ? a1 : 0.f;
}

// STRIDE: record stride; BLOB && bd >= 0: the 16 A rows are the OneBlob bins of dimension bd of a
// compact record (aoff unused).
template <bool PREC3, int STRIDE, bool BLOB>
__device__ __forceinline__ void dw_tile(const float* __restrict__ recs, int npts, int aoff,
                                        int boff, float (&acc)[4], int bd) {
  // acc[16 x 8] += sum_p A[p][aoff + m] * B[p][boff + n]; k-slot t <-> point 2t, t+4 <-> 2t+1
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll 2
  for (int k0 = 0; k0 < npts; k0 += 8) {
    const float* p0 = recs + (k0 + 2 * t) * STRIDE;
    const float* p1 = p0 + STRIDE;
    float va[4];
    if (BLOB && bd >= 0) {
      blob_dw_frag(p0, p1, bd, g, va);
    } else {
      va[0] = p0[aoff + g]; va[1] = p0[aoff + g + 8]; va[2] = p1[aoff + g]; va[3] = p1[aoff + g + 8];
    }
    FragA<PREC3> a;
    a.set(va);
    FragB<PREC3> b;
    b.set(p0[boff + g], p1[boff + g]);
    mma<PREC3>(acc, a, b);
  }
}

// The decoders for MT m-tiles of 16 records at wrec: h1, [geo, sdf], c1 and the rgb logits
// (RAW[0..2]; RAW[3] = sdf is the caller's).  Caller: one warp.
// COMPACT: the OneBlob A fragments are expanded from compact records.
template <bool PREC3, int MT, bool COMPACT, bool CG = false, bool CGF = false>
__device__ __forceinline__ void decoder_forward(float* __restrict__ wrec, const float* __restrict__ sw) {
  using L = Rec<COMPACT, CG, CGF>;
  constexpr int N = L::N;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  {  // h1 = relu([feat, blob] W0^T)
    float c[MT][4][4];
    zero_c(c);
    warp_gemm<10, 4, false, PREC3, N, COMPACT ? 4 : -1>(wrec, R_FEAT, sw + SW0, LD0, 0, 0, c);
    if (CGF) __syncwarp();  // h1 replaces feat: every lane has read its A fragments
    store_c<RELU, N>(wrec, L::H1, c);
  }
  __syncwarp();
  {  // [geo, sdf] = h1 W1^T
    float c[MT][2][4];
    zero_c(c);
    warp_gemm<4, 2, false, PREC3, N>(wrec, L::H1, sw + SW1, LD1, 0, 0, c);
    store_c<PLAIN, N>(wrec, L::GEO, c);
  }
  __syncwarp();
  {  // c1 = relu([blob, (cfeat,) geo, (sdf: zero weight row)] Wc0^T)
    float c[MT][4][4];
    zero_c(c);
    warp_gemm<Wts<CG>::KC, 4, false, PREC3, N, COMPACT ? 0 : -1>(wrec, COMPACT ? 0 : R_BLOB, sw + SWC0, LDC0, 0, 0, c);
    store_c<RELU, N>(wrec, L::C1, c);
  }
  __syncwarp();
  {  // rgb logits = c1 Wc1^T (cols 0..2 of an 8-wide tile)
    float c[MT][1][4];
    zero_c(c);
    warp_gemm<4, 1, false, PREC3, N>(wrec, L::C1, sw + Wts<CG>::SWC1, LDC1, 0, 0, c);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float* q0 = wrec + (mt * 16 + g) * N + L::RAW;
      if (t == 0) {
        q0[0] = c[mt][0][0]; q0[1] = c[mt][0][1];
        q0[8 * N] = c[mt][0][2]; q0[8 * N + 1] = c[mt][0][3];
      } else if (t == 1) {
        q0[2] = c[mt][0][0];
        q0[8 * N + 2] = c[mt][0][2];
      }
    }
  }
  __syncwarp();
}

// Zeroes the weight area, then stages the transposed decoder weights (zero padding included).
// Whole CTA; the caller synchronises before the first read.
template <bool CG = false>
__device__ __forceinline__ void stage_weights(float* __restrict__ sw, const Params& P) {
  using W = Wts<CG>;
  for (int q = threadIdx.x; q < W::TOTAL; q += blockDim.x) sw[q] = 0.f;
  __syncthreads();
  for (int q = threadIdx.x; q < 80 * 32; q += blockDim.x) {
    int i = q / 32, j = q % 32;
    sw[SW0 + i * LD0 + j] = P.w_sdf0[j * 80 + i];
  }
  for (int q = threadIdx.x; q < 32 * 16; q += blockDim.x) {
    int i = q / 16, jp = q % 16;  // jp: geo0..14 -> torch out 1..15, jp 15 -> out 0 (sdf)
    int jt = (jp + 1) & 15;
    sw[SW1 + i * LD1 + jp] = P.w_sdf1[jt * 32 + i];
  }
  for (int q = threadIdx.x; q < W::NC * 32; q += blockDim.x) {
    int i = q / 32, j = q % 32;
    sw[SWC0 + i * LDC0 + j] = P.w_col0[j * W::NC + i];
  }
  for (int q = threadIdx.x; q < 32 * 3; q += blockDim.x) {
    int i = q / 3, k = q % 3;
    sw[W::SWC1 + i * LDC1 + k] = P.w_col1[k * 32 + i];
  }
}

// loss normalisers of the gradient pass (batch-global counts n_fs, n_sdf, n_valid)
struct LossNorm {
  float fs_w = 0.f, sdf_w = 0.f, inv_nvalid = 0.f;
};
__device__ __forceinline__ LossNorm loss_norm(const int* __restrict__ counts) {
  LossNorm ln;
  const float n_fs = (float)counts[0], n_sdf = (float)counts[1];
  const float n = (float)(counts[0] + counts[1]);
  ln.fs_w = 1.0f - n_fs / n;
  ln.sdf_w = 1.0f - n_sdf / n;
  ln.inv_nvalid = 1.0f / (float)counts[2];
  return ln;
}

// Tile id of a weight-gradient layer whose tiles are [lo, hi) of the 42.  m-tile mt of the layer
// input covers its columns 16 mt .. 16 mt + 15 at record offset aoff; m-tiles
// [blob_mt, blob_mt + 3) are the OneBlob dimensions, read from the compact form.
template <bool PREC3, bool COMPACT, bool CG = false>
__device__ __forceinline__ void dw_layer_tile(const float* __restrict__ recs, int npts, int id,
                                              int lo, int aoff, int boff, int n_tiles_n,
                                              int blob_mt, float (&acc)[4]) {
  const int loc = id - lo, mt = loc / n_tiles_n, nt = loc % n_tiles_n;
  const int bd = (blob_mt >= 0 && mt >= blob_mt && mt < blob_mt + 3) ? mt - blob_mt : -1;
  dw_tile<PREC3, Rec<COMPACT, CG>::N, COMPACT>(recs, npts, aoff + 16 * mt, boff + 8 * nt, acc, bd);
}

// This warp's share of one weight-gradient layer: slot j holds tile w + j * nw.
template <bool PREC3, bool COMPACT, bool CG = false, int SLOTS>
__device__ __forceinline__ void dw_layer(const float* __restrict__ recs, int npts, int w, int nw,
                                         float (&acc)[SLOTS][4], int lo, int hi, int aoff,
                                         int boff, int n_tiles_n, int blob_mt) {
#pragma unroll
  for (int j = 0; j < SLOTS; ++j) {
    const int id = w + j * nw;
    if (id >= lo && id < hi)
      dw_layer_tile<PREC3, COMPACT, CG>(recs, npts, id, lo, aoff, boff, n_tiles_n, blob_mt, acc[j]);
  }
}

// Adds weight-gradient tile id (this lane's C fragment v; rows = in-feature, cols = out-unit) to
// the weight gradients in global memory.
template <bool CG = false>
__device__ __forceinline__ void dw_store(const Params& P, int id, const float (&v)[4]) {
  using W = Wts<CG>;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rloc = g + ((i & 2) ? 8 : 0), cloc = 2 * t + (i & 1);
    if (id < 2) {  // d w_col1 [3][32]
      const int in = 16 * id + rloc, out = cloc;
      if (out < 3) red_add(P.d_w_col1 + out * 32 + in, v[i]);
    } else if (id < W::SDF1_LO) {  // d w_col0 [32][NC]
      const int loc = id - 2, in = 16 * (loc / 4) + rloc, out = 8 * (loc % 4) + cloc;
      if (in < W::NC) red_add(P.d_w_col0 + out * W::NC + in, v[i]);
    } else if (id < W::SDF0_LO) {  // d w_sdf1 [16][32], stored column jp -> torch row (jp+1)&15
      const int loc = id - W::SDF1_LO, in = 16 * (loc / 2) + rloc, jp = 8 * (loc % 2) + cloc;
      red_add(P.d_w_sdf1 + ((jp + 1) & 15) * 32 + in, v[i]);
    } else {  // d w_sdf0 [32][80]
      const int loc = id - W::SDF0_LO, in = 16 * (loc / 4) + rloc, out = 8 * (loc % 4) + cloc;
      red_add(P.d_w_sdf0 + out * 80 + in, v[i]);
    }
  }
}

// d_rays_o / d_rays_d of ray rr (one warp): sums over its S records (rq) of d loss / d pts and
// z * d loss / d pts, parked in C1 slots 0..5
template <bool COMPACT, bool CG = false>
__device__ __forceinline__ void ray_grads(const Params& P, const float* __restrict__ rq, int rr,
                                          int lane) {
  float a[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int kk = lane; kk < P.S; kk += 32) {
    const float* rp = rq + (size_t)kk * Rec<COMPACT, CG>::N + Rec<COMPACT, CG>::C1;
#pragma unroll
    for (int d = 0; d < 6; ++d) a[d] += rp[d];
  }
#pragma unroll
  for (int d = 0; d < 6; ++d) a[d] = warp_sum(a[d]);
  if (lane == 0) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      if (P.d_rays_o) P.d_rays_o[rr * 3 + d] = a[d];
      if (P.d_rays_d) P.d_rays_d[rr * 3 + d] = a[3 + d];
    }
  }
}

// dgeo = dc1pre Wc0[:, 48:64] (colour grid: Wc0[:, 80:96]) -> dH = [dgeo(15), dsdf] in the GEO
// slots (SDF is the caller's), then dh1pre = (h1 > 0) * (dH W1) in place of h1; the caller's
// barrier and dW layer run between the two.  One warp, MT m-tiles.
template <bool PREC3, int MT, bool COMPACT, bool CG = false>
__device__ __forceinline__ void backward_geo(float* __restrict__ wrec, const float* __restrict__ sw) {
  using L = Rec<COMPACT, CG>;
  float c[MT][2][4];
  zero_c(c);
  warp_gemm<4, 2, true, PREC3, L::N>(wrec, L::C1, sw + SWC0, LDC0, 0, CG ? 80 : 48, c);
  store_c<PLAIN, L::N>(wrec, L::GEO, c);
}
template <bool PREC3, int MT, bool COMPACT, bool CG = false>
__device__ __forceinline__ void backward_h1(float* __restrict__ wrec, const float* __restrict__ sw) {
  using L = Rec<COMPACT, CG>;
  float c[MT][4][4];
  zero_c(c);
  warp_gemm<2, 4, true, PREC3, L::N>(wrec, L::GEO, sw + SW1, LD1, 0, 0, c);
  store_c<MASK, L::N>(wrec, L::H1, c);
}

// Phase 2 of both fused kernels for ray rr, one warp: the composite of its S samples (raw: the RAW
// slots of their records, stride N; zr: their z values), the per-ray outputs and, with BWD,
// d loss / d raw in RAW[0..3].  Per sample the five sigmoids are evaluated once: colours overwrite
// the rgb logits in RAW[0..2].  Lane owns samples kk = lane + 32 i, whose sigma(s/tr) and
// unnormalised weight u are kept
//   KPL > 0:  in registers, index i (the loops unroll over i < KPL; S <= 32 KPL);
//   KPL == 0: in the caller's shared arrays sg_s, u_s of S floats, index kk, in loops that are
//             not unrolled (the tile kernel: unrolled for its S <= 256 it is ~1400 instructions
//             longer and slower).
// Lane 0 hands the ray's loss partials to add_loss(term, v) (terms as in loss_acc: 0 rgb, 1 depth,
// only for rays with valid depth, 2 sdf, 3 fs) as soon as each is known, so that none stays live
// across the sample loops.
// (The RAW-slot pointer, rather than the record base, keeps k_fused_g at 96 registers and an
// 8-byte stack: with the record base, ptxas reloads a spilled address inside dw_tile's loop.)
// sdf2weights of one ray (one warp; samples, KPL and sg_r / u_r as in composite_ray): sg_r[j] =
// sigma(s/tr), u_r[j] = the unnormalised, truncated weight; returns the normaliser W (the weight
// of sample kk is u_r[j] / W).  COLOURS: also replace the rgb logits raw[kk*N + 0..2] by their
// sigmoids.  xrd_coslam_importance recomputes the coarse pass's weights through this function,
// so the pdf it samples comes from the weights that pass composited, bit for bit.
template <int N, int KPL, bool COLOURS>
__device__ __forceinline__ float composite_weights(float* raw, const float* zr, int S, float tr,
                                                   float* sg_r, float* u_r, int lane) {
  constexpr int UNROLL = KPL > 0 ? KPL : 1;
  const int n = KPL > 0 ? KPL : (S + 31) / 32;  // samples per lane
  int first = 0x7fffffff;
#pragma unroll UNROLL
  for (int i = 0; i < n; ++i) {
    const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
    if (KPL > 0) {
      sg_r[j] = 0.f;
      u_r[j] = 0.f;
    }
    if (kk < S) {
      float* rp = raw + kk * N;
      const float s = rp[3];
      const float sg = sigmoidf_acc(s / tr);
      sg_r[j] = sg;
      u_r[j] = sg * sigmoidf_acc((-s) / tr);
      if (COLOURS) {
        rp[0] = sigmoidf_acc(rp[0]);
        rp[1] = sigmoidf_acc(rp[1]);
        rp[2] = sigmoidf_acc(rp[2]);
      }
      if (kk < S - 1 && raw[(kk + 1) * N + 3] * s < 0.f) first = min(first, kk);
    }
  }
  first = warp_min_i(first);
  if (first == 0x7fffffff) first = 0;
  __syncwarp();
  const float zlim = zr[first] + tr;
  float usum = 0.f;
#pragma unroll UNROLL
  for (int i = 0; i < n; ++i) {
    const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
    if (kk < S) {
      const float u = (zr[kk] < zlim) ? u_r[j] : 0.f;
      u_r[j] = u;
      usum += u;
    }
  }
  usum = warp_sum(usum);
  return usum + 1e-8f;
}

template <int N, bool BWD, int KPL, typename AddLoss>
__device__ __forceinline__ void composite_ray(const Params& P, const LossNorm& ln, float* raw,
                                              const float* zr, float* sg_s, float* u_s, int rr,
                                              int lane, AddLoss add_loss) {
  constexpr int UNROLL = KPL > 0 ? KPL : 1;
  const int S = P.S;
  const int n = KPL > 0 ? KPL : (S + 31) / 32;  // samples per lane
  const float tr = P.trunc;
  float sg_reg[UNROLL], u_reg[UNROLL];
  float* sg_r = KPL > 0 ? sg_reg : sg_s;
  float* u_r = KPL > 0 ? u_reg : u_s;
  const float W = composite_weights<N, KPL, true>(raw, zr, S, tr, sg_r, u_r, lane);
  float o_r = 0.f, o_g = 0.f, o_b = 0.f, o_d = 0.f, o_acc = 0.f;
#pragma unroll UNROLL
  for (int i = 0; i < n; ++i) {
    const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
    if (kk < S) {
      const float* rp = raw + kk * N;
      const float w = u_r[j] / W;
      o_r = fmaf(w, rp[0], o_r);
      o_g = fmaf(w, rp[1], o_g);
      o_b = fmaf(w, rp[2], o_b);
      o_d = fmaf(w, zr[kk], o_d);
      o_acc += w;
    }
  }
  o_r = warp_sum(o_r); o_g = warp_sum(o_g); o_b = warp_sum(o_b);
  o_d = warp_sum(o_d); o_acc = warp_sum(o_acc);
  if (P.depth_var) {
    float v = 0.f;
#pragma unroll UNROLL
    for (int i = 0; i < n; ++i) {
      const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
      if (kk < S) {
        const float dz = zr[kk] - o_d;
        v = fmaf(u_r[j] / W, dz * dz, v);
      }
    }
    v = warp_sum(v);
    if (lane == 0) P.depth_var[rr] = v;
  }
  if (lane == 0) {
    if (P.rgb) { P.rgb[rr * 3] = o_r; P.rgb[rr * 3 + 1] = o_g; P.rgb[rr * 3 + 2] = o_b; }
    if (P.depth) P.depth[rr] = o_d;
    if (P.acc) P.acc[rr] = o_acc;
    if (P.disp) P.disp[rr] = 1.0f / fmaxf(1e-10f, o_d / o_acc);
  }
  if (BWD) {
    const float td = P.target_d[rr];
    const float tr_ = P.target_s[rr * 3], tg_ = P.target_s[rr * 3 + 1],
                tb_ = P.target_s[rr * 3 + 2];
    const bool valid = (td > 0.f) && (td < P.depth_trunc);
    const float RS = (float)P.Rg * (float)S;
    const float c_rgb = P.ls[0] * P.w_rgb * 2.0f / (3.0f * (float)P.Rg);
    const float g_r = c_rgb * (o_r - tr_), g_g = c_rgb * (o_g - tg_), g_b = c_rgb * (o_b - tb_);
    const float g_d = valid ? P.ls[1] * P.w_depth * 2.0f * (o_d - td) * ln.inv_nvalid : 0.f;
    if (lane == 0) {
      add_loss(0, (o_r - tr_) * (o_r - tr_) + (o_g - tg_) * (o_g - tg_) + (o_b - tb_) * (o_b - tb_));
      if (valid) add_loss(1, (o_d - td) * (o_d - td));
    }
    float qw = 0.f;
#pragma unroll UNROLL
    for (int i = 0; i < n; ++i) {
      const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
      if (kk < S) {
        const float* rp = raw + kk * N;
        const float q_ = g_r * rp[0] + g_g * rp[1] + g_b * rp[2] + g_d * zr[kk];
        qw = fmaf(q_, u_r[j] / W, qw);
      }
    }
    qw = warp_sum(qw);
    float a_fs = 0.f, a_sdf = 0.f;
    const float c_fs = P.ls[3] * P.w_fs * ln.fs_w * 2.0f / RS;
    const float c_sdf = P.ls[2] * P.w_sdf * ln.sdf_w * 2.0f / RS;
#pragma unroll UNROLL
    for (int i = 0; i < n; ++i) {
      const int kk = lane + 32 * i, j = KPL > 0 ? i : kk;
      if (kk >= S) continue;
      float* rp = raw + kk * N;
      const float z = zr[kk];
      const float s = rp[3];
      const float sg = sg_r[j];
      const float u = u_r[j];  // a * mask
      const float w = u / W;
      const float c0 = rp[0], c1 = rp[1], c2 = rp[2];
      const float q_ = g_r * c0 + g_g * c1 + g_b * c2 + g_d * z;
      float ds = (q_ - qw) / W * u * (1.f - 2.f * sg) / tr;
      const bool front = z < __fsub_rn(td, P.trunc);
      const bool back = z > __fadd_rn(td, P.trunc);
      if (front) {
        ds += c_fs * (s - 1.f);
        a_fs += (s - 1.f) * (s - 1.f);
      }
      if (!front && !back && td > 0.f) {
        float e = (z + s * P.trunc) - td;
        ds += c_sdf * e * P.trunc;
        a_sdf += e * e;
      }
      rp[0] = g_r * w * c0 * (1.f - c0);
      rp[1] = g_g * w * c1 * (1.f - c1);
      rp[2] = g_b * w * c2 * (1.f - c2);
      rp[3] = ds;
    }
    a_fs = warp_sum(a_fs);
    a_sdf = warp_sum(a_sdf);
    if (lane == 0) { add_loss(3, a_fs); add_loss(2, a_sdf); }
  }
}

// ----------------------------------------------------------------- fused ---
// The tile kernel's body; CG: with the colour grid (k_fused_c).
template <bool CG, bool BWD, bool PREC3, bool BPREC3, int SLOTS, typename PT>
__device__ __forceinline__ void fused_tile(const PT& P) {
  constexpr bool CGF = CG && !BWD;  // forward-only colour-grid pass: the compact record
  using L = Rec<false, CG, CGF>;
  using W = Wts<CG>;
  constexpr int REC = L::N;
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;                            // W::TOTAL
  float* recs = sw + W::TOTAL;                 // (blockDim.x + 8) * REC
  float* zbuf = recs + (blockDim.x + 8) * REC; // NR*S z values
  float* sgb = zbuf + P.NR * P.S;              // NR*S sigma(sdf/trunc)
  float* ub = sgb + P.NR * P.S;                // NR*S unnormalised weights
  float* xnb = ub + P.NR * P.S;                // NR*S*3 normalised coordinates
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nwarps = blockDim.x >> 5;
  const int S = P.S;

  __shared__ Lv s_lv[CG ? 2 * kL : kL];  // the colour grid's levels at kL
  load_levels(s_lv, P.g);
  if constexpr (CG) load_levels(s_lv + kL, P.gc);
  stage_weights<CG>(sw, P);
  // the 8 pad records after the tile stay zero for the whole kernel (k-step overrun of dw_tile)
  for (int q = tid; q < 8 * REC; q += blockDim.x) recs[blockDim.x * REC + q] = 0.f;
  const LossNorm ln = BWD ? loss_norm(P.counts) : LossNorm{};
  double l_sum[4] = {0.0, 0.0, 0.0, 0.0};  // loss sums of this thread (lane 0 of each warp)
  float dwacc[SLOTS][4];
#pragma unroll
  for (int j = 0; j < SLOTS; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) dwacc[j][i] = 0.f;
  __syncthreads();

  float* rec = recs + tid * REC;
  float* wrec = recs + (warp * 32) * REC;  // this warp's 32 records
  const bool need_dx = BWD && ((P.d_rays_o != nullptr) || (P.d_rays_d != nullptr));
  const bool map_grads = BWD && (P.d_table != nullptr);

  for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
    const int r0 = tile * P.NR;
    const int nr = min(P.NR, P.R - r0);
    const int npts = nr * S;
    const bool active = tid < npts;
    const bool warp_active = warp * 32 < npts;
    const int rl = active ? tid / S : 0;
    const int k = active ? tid - rl * S : 0;
    const int r = r0 + rl;
    float xn[3] = {0.f, 0.f, 0.f};
    float zv = 0.f;
    // ---------------- phase 1: forward -------------------------------------
    if (active) {
      zv = P.z_vals[(size_t)r * S + k];
      zbuf[tid] = zv;
      sample_xn(P, r, zv, xn);
#pragma unroll
      for (int d = 0; d < 3; ++d) xnb[tid * 3 + d] = xn[d];
      encode<1>(P.table, P.g.n_levels, s_lv, xn, rec, 0);
      if constexpr (CG) encode<1>(P.table_c, P.gc.n_levels, s_lv + kL, xn, rec + C_CFEAT, 0);
      blob_forward(xn, rec);
    } else {
      // inactive rows must read as zero in every GEMM (k-dimension of the dW tiles)
#pragma unroll 1
      for (int q = 0; q < REC; q += 4)
        *reinterpret_cast<float4*>(rec + q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    if (warp_active) decoder_forward<PREC3, 2, false, CG, CGF>(wrec, sw);
    if (active) {
      rec[L::RAW + 3] = rec[L::SDF];
      if (P.raw) {
        float4 rw = *reinterpret_cast<const float4*>(rec + L::RAW);
        *reinterpret_cast<float4*>(P.raw + ((size_t)r * S + k) * 4) = rw;
      }
    }
    __syncthreads();
    // ---------------- phase 2: per-ray composite, loss, d loss / d raw ----
    for (int q = warp; q < nr; q += nwarps)
      composite_ray<REC, BWD, 0>(P, ln, recs + (size_t)(q * S) * REC + L::RAW, zbuf + q * S,
                                 sgb + q * S, ub + q * S, r0 + q, lane,
                                 [&](int i, float v) { l_sum[i] += (double)v; });
    __syncthreads();
    if (!BWD) continue;
    // ---------------- phase 3: backward ----------------------------------
    // weight-gradient tiles owned by this warp: tile id = warp + j * nwarps
    auto dw_phase = [&](int lo, int hi, int aoff, int boff, int n_tiles_n, int blob_mt) {
      if (map_grads)
        dw_layer<BPREC3, false, CG>(recs, npts, warp, nwarps, dwacc, lo, hi, aoff, boff, n_tiles_n, blob_mt);
    };
    // d w_col1 += c1^T draw        (8-wide n tile over raw[4] + 4 floats of the next record:
    dw_phase(0, 2, L::C1, L::RAW, 1, -1);  //  columns 3..7 are never written out)
    __syncthreads();
    float draw3 = 0.f;
    if (active) {
      const float4 dr = *reinterpret_cast<const float4*>(rec + L::RAW);
      draw3 = dr.w;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float* w = sw + W::SWC1 + j * LDC1;
        const float c1 = rec[L::C1 + j];
        rec[L::C1 + j] = (c1 > 0.f) ? (dr.x * w[0] + dr.y * w[1] + dr.z * w[2]) : 0.f;
      }
    }
    __syncthreads();
    // d w_col0 += [blob, (cfeat,) geo, sdf]^T dc1pre   (row NC is discarded at write-out)
    dw_phase(2, W::SDF1_LO, R_BLOB, L::C1, 4, -1);
    __syncthreads();
    if (warp_active) backward_geo<BPREC3, 2, false, CG>(wrec, sw);
    if (CG && warp_active && (map_grads || need_dx)) {
      // dcfeat = dc1pre Wc0[:, 48:80] into the CFEAT slots (their last reader, the d w_col0
      // tiles, finished before the barrier above)
      float c[2][4][4];
      zero_c(c);
      warp_gemm<4, 4, true, BPREC3, REC>(wrec, L::C1, sw + SWC0, LDC0, 0, 48, c);
      store_c<PLAIN, REC>(wrec, C_CFEAT, c);
    }
    __syncwarp();
    if (active) rec[L::SDF] = draw3;
    __syncthreads();
    // d w_sdf1 += h1^T dH
    dw_phase(W::SDF1_LO, W::SDF0_LO, L::H1, L::GEO, 2, -1);
    __syncthreads();
    if (warp_active) backward_h1<BPREC3, 2, false, CG>(wrec, sw);
    __syncthreads();
    // d w_sdf0 += x^T dh1pre
    dw_phase(W::SDF0_LO, W::DW, R_FEAT, L::H1, 4, -1);
    // (readers of C1 / GEO slots are done: dW phases 2 and 3 finished before the last barrier)
    float hdx[2][2][3];  // hash-path d loss / d x for rows (mt, g / g+8), fragment layout
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) hdx[a][b][0] = hdx[a][b][1] = hdx[a][b][2] = 0.f;
    if (warp_active) {
      if (need_dx) {
        // dblob = dc1pre Wc0[:, 0:48] + dh1pre W0[:, 32:80]  -> scratch (C1 slots 0..31, GEO 32..47)
        float c[2][6][4];
        zero_c(c);
        warp_gemm<4, 6, true, BPREC3, REC>(wrec, L::C1, sw + SWC0, LDC0, 0, 0, c);
        warp_gemm<4, 6, true, BPREC3, REC>(wrec, L::H1, sw + SW0, LD0, 0, 32, c);
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 6; ++nt) {
            const int col = nt * 8 + 2 * t;
            const int off = (col < 32) ? (L::C1 + col) : (L::GEO + col - 32);
            float* q0 = wrec + (mt * 16 + g) * REC + off;
            *reinterpret_cast<float2*>(q0) = make_float2(c[mt][nt][0], c[mt][nt][1]);
            *reinterpret_cast<float2*>(q0 + 8 * REC) = make_float2(c[mt][nt][2], c[mt][nt][3]);
          }
      }
      if (map_grads || need_dx) {
        // dfeat = dh1pre W0[:, 0:32]; lane (g,t) holds (f0,f1) of level 4*nt+t for rows g, g+8
        float c[2][4][4];
        zero_c(c);
        warp_gemm<4, 4, true, BPREC3, REC>(wrec, L::H1, sw + SW0, LD0, 0, 0, c);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = warp * 32 + mt * 16 + g + 8 * h;
            if (row < npts) {
              const float x3[3] = {xnb[row * 3], xnb[row * 3 + 1], xnb[row * 3 + 2]};
              {  // the 4 levels of this lane (t, 4 + t, 8 + t, 12 + t) in one call
                LevelItems<4> it;
                bool any = false;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                  it.g[nt][0] = c[mt][nt][2 * h]; it.g[nt][1] = c[mt][nt][2 * h + 1];
                  it.on[nt] = (4 * nt + t) < P.g.n_levels && (it.g[nt][0] != 0.f || it.g[nt][1] != 0.f);
                  any |= it.on[nt];
                }
                if (any) {
                  const float3 d3 = hash_backward_multi<4>(P.table, P.d_table, s_lv, t, it, x3[0],
                                                           x3[1], x3[2], need_dx, map_grads);
                  hdx[mt][h][0] += d3.x; hdx[mt][h][1] += d3.y; hdx[mt][h][2] += d3.z;
                }
              }
              if constexpr (CG) {  // the colour grid: d loss / d cfeat of the same levels from CFEAT
                const float* cf = recs + row * REC + C_CFEAT;
                LevelItems<4> it;
                bool any = false;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                  const float2 gv = *reinterpret_cast<const float2*>(cf + 2 * (4 * nt + t));
                  it.g[nt][0] = gv.x; it.g[nt][1] = gv.y;
                  it.on[nt] = (4 * nt + t) < P.gc.n_levels && (gv.x != 0.f || gv.y != 0.f);
                  any |= it.on[nt];
                }
                if (any) {
                  const float3 d3 = hash_backward_multi<4>(P.table_c, P.d_table_c, s_lv + kL, t,
                                                           it, x3[0], x3[1], x3[2], need_dx,
                                                           map_grads);
                  hdx[mt][h][0] += d3.x; hdx[mt][h][1] += d3.y; hdx[mt][h][2] += d3.z;
                }
              }
            }
          }
      }
      if (need_dx) {
        // reduce the hash-path dx over the 4 lanes (t) that share a row, park it in RAW[0..2]
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int d = 0; d < 3; ++d) {
              float v = hdx[mt][h][d];
              v += __shfl_xor_sync(0xffffffffu, v, 1);
              v += __shfl_xor_sync(0xffffffffu, v, 2);
              if (t == 0) wrec[(mt * 16 + g + 8 * h) * REC + L::RAW + d] = v;
            }
        __syncwarp();
        if (active) {
          float dxn[3] = {rec[L::RAW], rec[L::RAW + 1], rec[L::RAW + 2]};
          blob_backward(xn, [&](int i) { return (i < 32) ? rec[L::C1 + i] : rec[L::GEO + i - 32]; }, dxn);
          // park d loss / d pts and z * d loss / d pts in the (dead) C1 slots 0..5
          float dp[3];
#pragma unroll
          for (int d = 0; d < 3; ++d)
            dp[d] = (float)((double)dxn[d] * P.g.binv[d]);
          rec[L::C1 + 0] = dp[0]; rec[L::C1 + 1] = dp[1]; rec[L::C1 + 2] = dp[2];
          rec[L::C1 + 3] = dp[0] * zv; rec[L::C1 + 4] = dp[1] * zv; rec[L::C1 + 5] = dp[2] * zv;
        }
      }
    }
    __syncthreads();
    if (need_dx) {
      for (int q = warp; q < nr; q += nwarps) ray_grads<false, CG>(P, recs + (size_t)(q * S) * REC, r0 + q, lane);
      __syncthreads();
    }
  }

  if (BWD) {
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (l_sum[i] != 0.0) atomicAdd(&P.loss_acc[i], l_sum[i]);
    }
    if (map_grads) {
#pragma unroll
      for (int j = 0; j < SLOTS; ++j) {
        const int id = warp + j * nwarps;
        if (id < W::DW) dw_store<CG>(P, id, dwacc[j]);
      }
    }
  }
}

template <bool BWD, bool PREC3, bool BPREC3, int SLOTS>
__global__ void __launch_bounds__(256) k_fused(const Params P) {
  fused_tile<false, BWD, PREC3, BPREC3, SLOTS>(P);
}
template <bool BWD, bool PREC3, bool BPREC3, int SLOTS>
__global__ void __launch_bounds__(256) k_fused_c(const ParamsC P) {
  fused_tile<true, BWD, PREC3, BPREC3, SLOTS>(P);
}


// ----------------------------------------------------------- fused, grouped ---
// v5: the same record-based algorithm, re-organised for latency hiding.  One persistent CTA
// per SM holds NGROUPS independent groups of 6 warps; a group owns GP record slots and pulls
// units of NR rays from a global queue, so at any time one group is in its gather phase
// (L1/L2 latency), another in the tensor-core phases and a third in the scatter phase: the
// phases that were serialised behind __syncthreads() in k_fused now overlap on the SM.
// Two threads share one sample point in the gather phases (8 levels each), one warp owns one
// 16-row MMA tile; all intra-group synchronisation is a named barrier (bar.sync grp+1, 192).
// Shared memory per slot: the 132-float compact record (GREC) and its z value; sigma(sdf/tr)
// and the composite weights live in registers (a lane owns <= G_KPL samples of a ray), xn is
// recomputed from the ray and z where the backward needs it.
constexpr int GT = 192;      // threads per group
constexpr int GW = 6;        // warps per group = m-tiles of 16 points per unit
constexpr int GP = 96;       // record slots per group
constexpr int NGROUPS = 3;
constexpr int G_SLOTS = 7;   // 42 weight-gradient tiles / 6 warps
constexpr int G_KPL = (GP + 31) / 32;  // samples per lane in the per-ray composite (S <= GP)
// Weight-gradient accumulators: warp gw's slot 0 (tile gw) stays in registers for the whole
// launch; tiles GW..41 are summed per CTA in shared memory, [tile - GW][4][32 lanes] (C-fragment
// order: conflict-free).  All 28 values per thread held in registers across the loop do not fit
// in 96 registers, and their spills to local memory compete with the gathers for L1.
constexpr int G_DWBUF = (DW_TILES - GW) * 4 * 32;  // floats
// dynamic shared memory: weights, NGROUPS x GP records + one z value per slot, and (gradient
// passes with map gradients) the weight-gradient buffer
constexpr size_t G_SMEM = sizeof(float) * ((size_t)SW_TOTAL + (size_t)NGROUPS * GP * (GREC + 1));
constexpr size_t G_SMEM_DW = G_SMEM + sizeof(float) * G_DWBUF;
// Stay in the 196 KB shared-memory configuration of an sm_90 SM (200 704 B): the next one up
// (228 KB) would cut the L1 the gathers rely on from ~60 KB to ~28 KB.  560 B: the kernel's
// static shared memory (s_lv, s_unit, s_loss); 1 KB: the per-CTA reservation.
static_assert(G_SMEM_DW + 560 + 1024 <= 196 * 1024, "k_fused_g outgrows the 196 KB carveout");

// Warp gw's share of one weight-gradient layer of k_fused_g (tiles gw + j GW in [lo, hi)): slot 0
// accumulates into dw0, every other tile into a zeroed fragment that is then added to dwbuf (the
// NGROUPS groups add to the same tiles).
template <bool PREC3>
__device__ __forceinline__ void dw_layer_g(const float* __restrict__ recs, int npts, int gw,
                                           float (&dw0)[4], float* __restrict__ dwbuf, int lo,
                                           int hi, int aoff, int boff, int n_tiles_n, int blob_mt) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < G_SLOTS; ++j) {
    const int id = gw + j * GW;
    if (id < lo || id >= hi) continue;
    if (j == 0) {
      dw_layer_tile<PREC3, true>(recs, npts, id, lo, aoff, boff, n_tiles_n, blob_mt, dw0);
    } else {
      float c[4] = {0.f, 0.f, 0.f, 0.f};
      dw_layer_tile<PREC3, true>(recs, npts, id, lo, aoff, boff, n_tiles_n, blob_mt, c);
      float* q = dwbuf + (id - GW) * 4 * 32 + lane;
#pragma unroll
      for (int i = 0; i < 4; ++i) atomicAdd(q + 32 * i, c[i]);
    }
  }
}

__device__ __forceinline__ void group_sync(int grp) {
  asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(GT) : "memory");
}

template <bool BWD, bool PREC3, bool BPREC3>
__global__ void __launch_bounds__(GT * NGROUPS, 1) k_fused_g(const Params P, int* __restrict__ queue) {
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;  // SW_TOTAL
  const int tid = threadIdx.x;
  const int grp = tid / GT, gt = tid - grp * GT;
  const int gw = gt >> 5, lane = gt & 31;
  float* recs = sw + SW_TOTAL + grp * (GP * GREC);
  float* zbuf = sw + SW_TOTAL + NGROUPS * (GP * GREC) + grp * GP;  // GP z values
  float* dwbuf = sw + G_SMEM / sizeof(float);  // G_DWBUF, only when map_grads
  const int S = P.S;
  const bool need_dx = BWD && ((P.d_rays_o != nullptr) || (P.d_rays_d != nullptr));
  const bool map_grads = BWD && (P.d_table != nullptr);

  __shared__ Lv s_lv[kL];
  __shared__ int s_unit[NGROUPS];
  __shared__ double s_loss[4];  // loss sums of the CTA (registers are the scarce resource here)
  load_levels(s_lv, P.g);
  if (tid < 4) s_loss[tid] = 0.0;
  for (int q = gt; q < GP * GREC; q += GT) recs[q] = 0.f;
  if (map_grads)
    for (int q = tid; q < G_DWBUF; q += blockDim.x) dwbuf[q] = 0.f;
  stage_weights(sw, P);
  const LossNorm ln = BWD ? loss_norm(P.counts) : LossNorm{};
  float dw0[4] = {0.f, 0.f, 0.f, 0.f};  // weight-gradient tile gw
  __syncthreads();

  const int p = gt >> 1, half = gt & 1;       // gather phases: two threads per point
  float* rec = recs + p * GREC;
  float* wrec = recs + (gw * 16) * GREC;      // MMA phases: this warp's 16 records
  int prev_npts = 0;

  for (;;) {
    if (gt == 0) s_unit[grp] = atomicAdd(queue, 1);
    group_sync(grp);  // also: every reader of the previous unit's records is done
    const int unit = s_unit[grp];
    if (unit >= P.n_tiles) break;
    const int r0 = unit * P.NR;
    const int nr = min(P.NR, P.R - r0);
    const int npts = nr * S;
    const bool active = p < npts;
    const bool warp_active = gw * 16 < npts;
    const int rl = active ? p / S : 0;
    const int k = active ? p - rl * S : 0;
    const int r = r0 + rl;
    float xn[3] = {0.f, 0.f, 0.f};
    float zv = 0.f;
    // ---------------- phase 1: forward -------------------------------------
    if (active) {
      zv = P.z_vals[(size_t)r * S + k];
      sample_xn(P, r, zv, xn);
      if (half == 0) zbuf[p] = zv;
      encode<2>(P.table, P.g.n_levels, s_lv, xn, rec, half);
      // OneBlob dims 0, 1 (half 0) and 2 (half 1); constant indices keep xn in registers
      if (half) {
        blob_compact_dim(xn[2], rec + G_BLOB + 8, reinterpret_cast<uint8_t*>(rec + G_BLOB + 14));
      } else {
        blob_compact_dim(xn[0], rec + G_BLOB, reinterpret_cast<uint8_t*>(rec + G_BLOB + 12));
        blob_compact_dim(xn[1], rec + G_BLOB + 4, reinterpret_cast<uint8_t*>(rec + G_BLOB + 13));
      }
    } else if (p < prev_npts) {
      // rows left dirty by a larger unit must read as zero in every GEMM
      float* z0 = rec + half * (GREC / 2);
#pragma unroll 1
      for (int q = 0; q < GREC / 2; q += 2) *reinterpret_cast<float2*>(z0 + q) = make_float2(0.f, 0.f);
    }
    prev_npts = npts;
    __syncwarp();
    if (warp_active) decoder_forward<PREC3, 1, true>(wrec, sw);
    if (active && half == 0) {
      rec[G_RAW + 3] = rec[G_SDF];
      if (P.raw) {
        float4 rw = *reinterpret_cast<const float4*>(rec + G_RAW);
        *reinterpret_cast<float4*>(P.raw + ((size_t)r * S + k) * 4) = rw;
      }
    }
    group_sync(grp);
    // ---------------- phase 2: per-ray composite, loss, d loss / d raw ----
    for (int q = gw; q < nr; q += GW)
      composite_ray<GREC, BWD, G_KPL>(P, ln, recs + (size_t)(q * S) * GREC + G_RAW, zbuf + q * S,
                                      nullptr, nullptr, r0 + q, lane,
                                      [&](int i, float v) { atomicAdd(&s_loss[i], (double)v); });
    if (!BWD) continue;  // the barrier at the top of the loop orders the next unit
    group_sync(grp);
    // ---------------- phase 3: backward ----------------------------------
    auto dw_phase = [&](int lo, int hi, int aoff, int boff, int n_tiles_n, int blob_mt) {
      if (map_grads)
        dw_layer_g<BPREC3>(recs, npts, gw, dw0, dwbuf, lo, hi, aoff, boff, n_tiles_n, blob_mt);
    };
    // d w_col1 += c1^T draw   (8-wide n tile over raw[4] + 4 floats of the next record: columns
    dw_phase(0, 2, G_C1, G_RAW, 1, -1);  //  3..7 are never written out; the last record's
    group_sync(grp);                     //  overrun stays inside the kernel's shared memory)
    float draw3 = 0.f;
    if (active) {
      const float4 dr = *reinterpret_cast<const float4*>(rec + G_RAW);
      draw3 = dr.w;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int j = half * 16 + jj;
        const float* w = sw + SWC1 + j * LDC1;
        const float c1 = rec[G_C1 + j];
        rec[G_C1 + j] = (c1 > 0.f) ? (dr.x * w[0] + dr.y * w[1] + dr.z * w[2]) : 0.f;
      }
    }
    group_sync(grp);
    // d w_col0 += [blob, geo, sdf]^T dc1pre   (row 63 is discarded at write-out)
    dw_phase(2, 18, 0, G_C1, 4, 0);
    group_sync(grp);
    if (warp_active) backward_geo<BPREC3, 1, true>(wrec, sw);
    __syncwarp();
    if (active && half == 0) rec[G_SDF] = draw3;
    group_sync(grp);
    // d w_sdf1 += h1^T dH
    dw_phase(18, 22, G_H1, G_GEO, 2, -1);
    group_sync(grp);
    if (warp_active) backward_h1<BPREC3, 1, true>(wrec, sw);
    group_sync(grp);
    // d w_sdf0 += x^T dh1pre
    dw_phase(22, 42, G_FEAT, G_H1, 4, 2);
    // (readers of C1 / GEO slots are done: dW phases 2 and 3 finished before the last barrier)
    float cfeat[1][4][4];
    zero_c(cfeat);
    if (warp_active) {
      if (need_dx) {
        // dblob = dc1pre Wc0[:, 0:48] + dh1pre W0[:, 32:80]  -> scratch (C1 slots 0..31, GEO 32..47)
        // in two passes (register budget): columns 32..47 go to the dead GEO slots at once,
        // columns 0..31 replace dc1pre after the last read of it
        {
          float c[1][2][4];
          zero_c(c);
          warp_gemm<4, 2, true, BPREC3, GREC>(wrec, G_C1, sw + SWC0, LDC0, 0, 32, c);
          warp_gemm<4, 2, true, BPREC3, GREC>(wrec, G_H1, sw + SW0, LD0, 0, 64, c);
          store_c<PLAIN, GREC>(wrec, G_GEO, c);
        }
        {
          float c[1][4][4];
          zero_c(c);
          warp_gemm<4, 4, true, BPREC3, GREC>(wrec, G_C1, sw + SWC0, LDC0, 0, 0, c);
          warp_gemm<4, 4, true, BPREC3, GREC>(wrec, G_H1, sw + SW0, LD0, 0, 32, c);
          __syncwarp();
          store_c<PLAIN, GREC>(wrec, G_C1, c);
        }
      }
      // dfeat = dh1pre W0[:, 0:32]
      if (map_grads || need_dx) warp_gemm<4, 4, true, BPREC3, GREC>(wrec, G_H1, sw + SW0, LD0, 0, 0, cfeat);
    }
    group_sync(grp);  // every warp is past the x^T dh1pre tiles: the FEAT slots are free
    if (warp_active && (map_grads || need_dx)) store_c<PLAIN, GREC>(wrec, G_FEAT, cfeat);
    group_sync(grp);
    // ---- hash backward, point-parallel and BALANCED: thread (pp, half) owns levels half, half+2, ..
    // of point pp = every 6th point of the unit per warp (a ray's samples behind the surface carry
    // no gradient: ray-major assignment would leave whole warps idle).  d loss / d xn comes from
    // a second gather of the corners; the table gradient is scattered in corner pairs.
    {
      const int qd = gt >> 1;
      const int pp = (qd & 15) * GW + (qd >> 4);
      const bool act2 = pp < npts;
      float* rec2 = recs + pp * GREC;
      float dxh[3] = {0.f, 0.f, 0.f};
      float xq[3] = {0.f, 0.f, 0.f};
      const float zq = act2 ? zbuf[pp] : 0.f;
      if (act2) sample_xn(P, r0 + pp / S, zq, xq);  // xn of point pp, exactly as in the forward
      if (act2 && (map_grads || need_dx)) {
#pragma unroll 1
        for (int i2 = 0; i2 < kL / 2; i2 += 2) {  // two levels per call: half + 2 i2, half + 2 i2 + 2
          LevelItems<2> it;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int l = half + 2 * (i2 + e);
            const float2 gv = *reinterpret_cast<const float2*>(rec2 + G_FEAT + 2 * l);
            it.g[e][0] = gv.x; it.g[e][1] = gv.y;
            it.on[e] = l < P.g.n_levels && (gv.x != 0.f || gv.y != 0.f);
          }
          if (it.on[0] || it.on[1]) {
            const float3 d3 = hash_backward_multi<2>(P.table, P.d_table, s_lv, half + 2 * i2, it,
                                                     xq[0], xq[1], xq[2], need_dx,
                                                     map_grads, 2);
            dxh[0] += d3.x; dxh[1] += d3.y; dxh[2] += d3.z;
          }
        }
      }
      if (need_dx) {
        // the two halves of a point are adjacent lanes: sum their level shares
#pragma unroll
        for (int d = 0; d < 3; ++d) dxh[d] += __shfl_xor_sync(0xffffffffu, dxh[d], 1);
        float dp0 = 0.f, dp1 = 0.f;
        if (act2) {
          auto dblob = [&](int i) { return (i < 32) ? rec2[G_C1 + i] : rec2[G_GEO + i - 32]; };
          if (half == 0) {
            dp0 = (float)((double)(blob_backward_dim(xq[0], 0, dblob) + dxh[0]) * P.g.binv[0]);
            dp1 = (float)((double)(blob_backward_dim(xq[1], 1, dblob) + dxh[1]) * P.g.binv[1]);
          } else {
            dp0 = (float)((double)(blob_backward_dim(xq[2], 2, dblob) + dxh[2]) * P.g.binv[2]);
          }
        }
        __syncwarp();  // both halves have read the dblob scratch before C1[0..5] is reused
        if (act2) {
          // park d loss / d pts and z * d loss / d pts in the (dead) C1 slots 0..5
          if (half == 0) {
            rec2[G_C1 + 0] = dp0; rec2[G_C1 + 3] = dp0 * zq;
            rec2[G_C1 + 1] = dp1; rec2[G_C1 + 4] = dp1 * zq;
          } else {
            rec2[G_C1 + 2] = dp0; rec2[G_C1 + 5] = dp0 * zq;
          }
        }
      }
    }
    if (need_dx) {
      group_sync(grp);
      for (int q = gw; q < nr; q += GW) ray_grads<true>(P, recs + (size_t)(q * S) * GREC, r0 + q, lane);
    }
  }

  if (BWD) {
    __syncthreads();
    if (tid < 4 && s_loss[tid] != 0.0) atomicAdd(&P.loss_acc[tid], s_loss[tid]);
    if (map_grads) {
      // the groups' register tiles 0..GW-1 go through the (dead) record area, [grp][tile][4][32];
      // then one warp per tile and one red.global per element and CTA
      float* red = sw + SW_TOTAL;
#pragma unroll
      for (int i = 0; i < 4; ++i) red[((grp * GW + gw) * 4 + i) * 32 + lane] = dw0[i];
      __syncthreads();
      for (int id = tid >> 5; id < DW_TILES; id += NGROUPS * GW) {
        float v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (id < GW) {
            v[i] = red[(id * 4 + i) * 32 + lane];
            for (int gs = 1; gs < NGROUPS; ++gs) v[i] += red[((gs * GW + id) * 4 + i) * 32 + lane];
          } else {
            v[i] = dwbuf[(id - GW) * 4 * 32 + 32 * i + lane];
          }
        }
        dw_store(P, id, v);
      }
    }
  }
}

struct FinalizeParams {
  const double* loss_acc;
  const int* counts;
  float* losses;
  int R, S;
  float w_rgb, w_depth, w_sdf, w_fs;
};

__global__ void k_finalize(FinalizeParams p) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float n_fs = (float)p.counts[0], n_sdf = (float)p.counts[1];
  const float n = (float)(p.counts[0] + p.counts[1]);
  const float fs_w = 1.0f - n_fs / n, sdf_w = 1.0f - n_sdf / n;
  const double RS = (double)p.R * (double)p.S;
  p.losses[0] = (float)(p.loss_acc[0] / (3.0 * p.R)) * p.w_rgb;
  p.losses[1] = (float)(p.loss_acc[1] / (double)p.counts[2]) * p.w_depth;  // NaN if no valid depth, like torch
  p.losses[2] = (float)(p.loss_acc[2] / RS) * sdf_w * p.w_sdf;
  p.losses[3] = (float)(p.loss_acc[3] / RS) * fs_w * p.w_fs;
}

// ------------------------------------------------------------- smoothness ---
// One CTA per (level, slab of kSmoothPlanes x planes of the n^3 lattice).  It sweeps its planes
// with a window of plane features in shared memory: plane x sits in slot x & 3, so the plane
// written in one step (x + 1) never overwrites one the previous step still reads (x - 2 is its
// oldest) and one __syncthreads per plane suffices.  A slab recomputes the features of its two
// boundary planes instead of reading them from a lattice-sized buffer.
//
// The lattice is axis-aligned, so a point's cell and weight along an axis depend only on its
// index along that axis, and the cells a slab touches form a box.  Where that box of table
// entries fits in shared memory (the coarse levels, where many points share a cell) the CTA
// loads it once and interpolates from it, and gathers the gradient per vertex: plane x adds to
// the two vertex planes of its x cell, and each (y, z) vertex sums the points of the rows whose
// cells touch it (no atomics).  The box leaves with one reduction per touched x pair of entries.
// Elsewhere each point gathers its 8 corners and scatters to them.
constexpr int kSmoothThreads = 512, kSmoothPlanes = 4, kSmoothMaxN = 75;  // 5 n^2 float2 fit
// entries of the shared-memory box (table values + gradient: 16 B each), at most
constexpr int kSmoothBox = 9216;

struct SmoothHdr {
  double loss_acc;
  unsigned int done;  // CTAs that have added their part of the loss
};

struct SmoothParams {
  GridDev g;
  const float* table;
  int n;  // lattice side (sample_points - 1)
  double voxel, off[3], rnd[3];
  const float* rand_dev;  // DEVICE [6] overriding off/rnd (graph replay)
  double offmax[3], margin;
  float* d_table;
  SmoothHdr* hdr;
  float* loss;
  float coef;        // grad_scale * weight / sample_points^3
  float loss_scale;  // weight / sample_points^3
  int box_cap;       // entries of the shared-memory box this launch has room for
};

// normalised coordinate of lattice index i along axis d
__device__ __forceinline__ float smooth_xn(const SmoothParams& p, int d, int i) {
  // pts = (coords + rand) * voxel + bb_min + offset ; then (pts - bb_min)/(bb_max-bb_min), all f64
  const double rnd = p.rand_dev ? (double)p.rand_dev[3 + d] : p.rnd[d];
  const double off = p.rand_dev ? (double)p.rand_dev[d] * p.offmax[d] + p.margin : p.off[d];
  const double pt = ((double)(float)i + rnd) * p.voxel + p.g.bmin[d] + off;
  return (float)((pt - p.g.bmin[d]) / (p.g.bmax[d] - p.g.bmin[d]));
}

// first i in [0, n) with c[i] >= v, n if none (c nondecreasing)
__device__ __forceinline__ int first_ge(const int* c, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (c[m] < v) lo = m + 1; else hi = m;
  }
  return lo;
}

// Features of one level over the lattice, the squared differences of neighbours (each counted
// once, from its upper end) and, with d_table, their gradient added to the table.  The last CTA
// to finish writes loss = loss_scale * sum.  Launched with kSmoothThreads threads and
// (5 n^2 + 2 box_cap) float2 of dynamic shared memory.
__global__ void __launch_bounds__(kSmoothThreads) k_smooth_bwd(SmoothParams p) {
  extern __shared__ float2 s_win[];  // 4 slots of n^2 features | n^2 point gradients | box | box
  __shared__ float s_xn[3][kSmoothMaxN], s_w[3][kSmoothMaxN];
  __shared__ uint32_t s_cell[3][kSmoothMaxN];
  __shared__ int s_c[3][kSmoothMaxN];  // cell relative to the box
  __shared__ float s_part[kSmoothThreads / 32];
  __shared__ bool s_last;
  const int n = p.n, nn = n * n, l = blockIdx.y;
  Lv L;
  L.scale = p.g.scale[l]; L.res = p.g.res[l]; L.size = p.g.size[l]; L.offset = p.g.offset[l];
  L.hashed = p.g.hashed[l]; L.magic = p.g.magic[l];
  for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) {
    const int d = i / n, j = i % n;
    const float xn = smooth_xn(p, d, j);
    s_xn[d][j] = xn;
    pos_fract(xn, L.scale, s_w[d][j], s_cell[d][j]);
  }
  __syncthreads();
  const int x0 = blockIdx.x * kSmoothPlanes, x1 = min(x0 + kSmoothPlanes, n);
  // the box: cells of planes x0 - 1 .. x1 and of all rows, plus their upper vertex; an even
  // number of x vertices so that the box leaves in x pairs
  const uint32_t org[3] = {s_cell[0][max(x0 - 1, 0)], s_cell[1][0], s_cell[2][0]};
  const int B0 = ((int)(s_cell[0][min(x1, n - 1)] - org[0]) + 3) & ~1;
  const int B1 = (int)(s_cell[1][n - 1] - org[1]) + 2, B2 = (int)(s_cell[2][n - 1] - org[2]) + 2;
  const bool box = (long long)B0 * B1 * B2 <= p.box_cap;
  const bool box_grad = box && p.d_table;
  const float2* __restrict__ tab = reinterpret_cast<const float2*>(p.table);
  float2* s_g = s_win + 4 * nn;
  float2* s_tab = s_g + nn;
  float2* s_acc = s_tab + p.box_cap;
  if (box) {
    for (int i = threadIdx.x; i < 3 * n; i += blockDim.x)
      s_c[i / n][i % n] = (int)(s_cell[i / n][i % n] - org[i / n]);
    for (int e = threadIdx.x; e < B0 * B1 * B2; e += blockDim.x) {
      const int a = e % B0, b = (e / B0) % B1, c = e / (B0 * B1);
      s_tab[e] = __ldg(&tab[grid_index(L, org[0] + a, org[1] + b, org[2] + c)]);
      if (box_grad) s_acc[e] = make_float2(0.f, 0.f);
    }
    __syncthreads();
  }
  auto plane = [&](int x) {
    float2* s = s_win + (x & 3) * nn;
    for (int q = threadIdx.x; q < nn; q += blockDim.x) {
      const int iy = q / n, iz = q % n;
      if (box) {  // level_feature's arithmetic on the box
        const float w[3] = {s_w[0][x], s_w[1][iy], s_w[2][iz]};
        const float2* v = s_tab + s_c[0][x] + B0 * (s_c[1][iy] + B1 * s_c[2][iz]);
        float f0 = 0.f, f1 = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float wk = ((k & 1) ? w[0] : 1.f - w[0]) * ((k & 2) ? w[1] : 1.f - w[1]) *
                           ((k & 4) ? w[2] : 1.f - w[2]);
          const float2 vk = v[(k & 1) + ((k >> 1) & 1) * B0 + (k >> 2) * B0 * B1];
          f0 = fmaf(wk, vk.x, f0);
          f1 = fmaf(wk, vk.y, f1);
        }
        s[q] = make_float2(f0, f1);
      } else {
        const float xn[3] = {s_xn[0][x], s_xn[1][iy], s_xn[2][iz]};
        s[q] = level_feature(p.table, L, xn);
      }
    }
  };
  if (x0 > 0) plane(x0 - 1);
  plane(x0);
  float part = 0.f;
  for (int x = x0; x < x1; ++x) {
    if (x + 1 < n) plane(x + 1);
    __syncthreads();
    const float2* F = s_win + (x & 3) * nn;
    const float2* nb[3][2] = {{s_win + ((x - 1) & 3) * nn, s_win + ((x + 1) & 3) * nn},
                              {F - n, F + n}, {F - 1, F + 1}};
    for (int q = threadIdx.x; q < nn; q += blockDim.x) {
      const int iy = q / n, iz = q % n;
      const int ci[3] = {x, iy, iz};
      const float2 f = F[q];
      float g0 = 0.f, g1 = 0.f;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        if (ci[d] > 0) {
          const float2 o = nb[d][0][q];
          const float a = f.x - o.x, b = f.y - o.y;
          g0 += a; g1 += b;
          part += a * a + b * b;
        }
        if (ci[d] < n - 1) {
          const float2 o = nb[d][1][q];
          g0 -= o.x - f.x; g1 -= o.y - f.y;
        }
      }
      if (!p.d_table) continue;
      g0 *= 2.f * p.coef; g1 *= 2.f * p.coef;
      if (box) {
        s_g[q] = make_float2(g0, g1);
      } else {
        const float xn[3] = {s_xn[0][x], s_xn[1][iy], s_xn[2][iz]};
        float w[3];
        uint32_t c[3], idx[8];
        for (int d = 0; d < 3; ++d) pos_fract(xn[d], L.scale, w[d], c[d]);
        corner_indices(L, c, idx);
        scatter_corners(p.d_table, idx, w, g0, g1);
      }
    }
    if (box_grad) {
      // (y, z) vertex (b, c) of plane x's two x vertices: the points of rows j with
      // s_c[1][j] in {b - 1, b} and columns k with s_c[2][k] in {c - 1, c}
      __syncthreads();
      const float wx = s_w[0][x];
      float2* t = s_acc + s_c[0][x];
      for (int v = threadIdx.x; v < B1 * B2; v += blockDim.x) {
        const int b = v % B1, c = v / B1;
        const int j0 = first_ge(s_c[1], n, b - 1), j1 = first_ge(s_c[1], n, b + 1);
        const int k0 = first_ge(s_c[2], n, c - 1), k1 = first_ge(s_c[2], n, c + 1);
        float a0 = 0.f, a1 = 0.f;
        for (int j = j0; j < j1; ++j) {
          const float wy = s_c[1][j] == b ? 1.f - s_w[1][j] : s_w[1][j];
          for (int k = k0; k < k1; ++k) {
            const float wyz = wy * (s_c[2][k] == c ? 1.f - s_w[2][k] : s_w[2][k]);
            const float2 g = s_g[j * n + k];
            a0 = fmaf(wyz, g.x, a0);
            a1 = fmaf(wyz, g.y, a1);
          }
        }
        if (a0 != 0.f || a1 != 0.f) {
          float2* e = t + B0 * v;
          e[0].x += (1.f - wx) * a0; e[0].y += (1.f - wx) * a1;
          e[1].x += wx * a0; e[1].y += wx * a1;
        }
      }
    }
  }
  if (box_grad) {
    __syncthreads();
    for (int e = 2 * threadIdx.x; e < B0 * B1 * B2; e += 2 * blockDim.x) {
      const float2 lo = s_acc[e], hi = s_acc[e + 1];
      if (lo.x == 0.f && lo.y == 0.f && hi.x == 0.f && hi.y == 0.f) continue;
      const int a = e % B0, b = (e / B0) % B1, c = e / (B0 * B1);
      scatter_corner_pair(p.d_table, grid_index(L, org[0] + a, org[1] + b, org[2] + c),
                          grid_index(L, org[0] + a + 1, org[1] + b, org[2] + c), lo, hi);
    }
  }
  // one double atomic per CTA; the last CTA (ticket after a fence) writes the loss
  part = warp_sum(part);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < kSmoothThreads / 32; ++i) a += (double)s_part[i];
    if (a != 0.0) atomicAdd(&p.hdr->loss_acc, a);
    __threadfence();
    s_last = atomicAdd(&p.hdr->done, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    p.loss[0] = (float)(*(volatile double*)&p.hdr->loss_acc * (double)p.loss_scale);
  }
}

// hash encode only
__global__ void __launch_bounds__(256) k_encode(GridDev g, const float* table, const float* x,
                                                int n, float* feat, uint32_t* idx_out) {
  __shared__ Lv s_lv[kL];
  load_levels(s_lv, g);
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int pt = q / kL, l = q % kL;
  if (pt >= n || l >= g.n_levels) return;
  const Lv L = s_lv[l];
  const float xn[3] = {x[pt * 3], x[pt * 3 + 1], x[pt * 3 + 2]};
  if (idx_out) {
    float w[3];
    uint32_t c[3], idx[8];
    for (int d = 0; d < 3; ++d) pos_fract(xn[d], L.scale, w[d], c[d]);
    corner_indices(L, c, idx);
#pragma unroll
    for (int k = 0; k < 8; ++k) idx_out[((size_t)pt * g.n_levels + l) * 8 + k] = idx[k];
  }
  if (feat) {
    const float2 f = level_feature(table, L, xn);
    feat[(size_t)pt * 2 * g.n_levels + 2 * l] = f.x;
    feat[(size_t)pt * 2 * g.n_levels + 2 * l + 1] = f.y;
  }
}

// ------------------------------------------------------- point queries (mesher) ---
// query_color_sdf / query_sdf at arbitrary points (joint_encoding.py:425-481): thread per point,
// hash + OneBlob encoding into a shared-memory record, the two decoders in plain fp32 FMAs
// (the mesher path is not hot; exact fp32 keeps it within 1e-6 of the oracle).
struct QueryParams {
  GridDev g;
  const float* table;
  const float *w_sdf0, *w_sdf1, *w_col0, *w_col1;
  const float* pts;   // [P,3]
  int P, normalised;  // normalised = 1: pts are already (p - min) / (max - min)
  float* raw;         // [P,4] rgb logits ++ sdf, or NULL
  float* geo;         // [P,15] or NULL
  float* feat;        // [P,32] hash features (query_sdf(embed=True)) or NULL
};
// k_query_c: the colour grid on top (normalised coordinates come from g's bound)
struct QueryParamsC : QueryParams {
  GridDev gc;
  const float* table_c;
};

// The query kernel's body; CG: with the colour grid (k_query_c, ColorSDFNet).
template <bool CG, typename QT>
__device__ __forceinline__ void query_points(const QT& Q) {
  constexpr int NC = Wts<CG>::NC;
  extern __shared__ __align__(16) float qrec[];  // 128 records
  __shared__ Lv s_lv[CG ? 2 * kL : kL];  // the colour grid's levels at kL
  load_levels(s_lv, Q.g);
  if constexpr (CG) load_levels(s_lv + kL, Q.gc);
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Q.P) return;
  float* rec = qrec + threadIdx.x * Rec<false, CG>::N;
  float xn[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float v = Q.pts[(size_t)p * 3 + d];
    xn[d] = Q.normalised ? v : normalise(v, Q.g.bmin[d], Q.g.bmax[d]);
  }
  encode<1>(Q.table, Q.g.n_levels, s_lv, xn, rec, 0);
  if constexpr (CG) encode<1>(Q.table_c, Q.gc.n_levels, s_lv + kL, xn, rec + C_CFEAT, 0);
  blob_forward(xn, rec);
  if (Q.feat)
#pragma unroll 4
    for (int j = 0; j < 32; ++j) Q.feat[(size_t)p * 32 + j] = rec[R_FEAT + j];
  if (!Q.raw && !Q.geo) return;
  // h1 = relu(W0 [feat, blob]);  [sdf, geo] = W1 h1  (torch rows: 0 = sdf, 1..15 = geo)
  float h1[32];
#pragma unroll 1
  for (int j = 0; j < 32; ++j) {
    float a = 0.f;
    const float* w = Q.w_sdf0 + j * 80;
    for (int i = 0; i < 80; ++i) a = fmaf(__ldg(w + i), rec[R_FEAT + i], a);  // FEAT|BLOB contiguous
    h1[j] = fmaxf(a, 0.f);
  }
  float so[16];
#pragma unroll 1
  for (int j = 0; j < 16; ++j) {
    float a = 0.f;
    const float* w = Q.w_sdf1 + j * 32;
#pragma unroll
    for (int i = 0; i < 32; ++i) a = fmaf(__ldg(w + i), h1[i], a);
    so[j] = a;
  }
  if (Q.geo)
    for (int j = 0; j < 15; ++j) Q.geo[(size_t)p * 15 + j] = so[1 + j];
  if (!Q.raw) return;
  // colour: c1 = relu(Wc0 [blob, (cfeat,) geo]);  rgb logits = Wc1 c1
  float c1[32];
#pragma unroll 1
  for (int j = 0; j < 32; ++j) {
    float a = 0.f;
    const float* w = Q.w_col0 + j * NC;
    for (int i = 0; i < 48; ++i) a = fmaf(__ldg(w + i), rec[R_BLOB + i], a);
    if constexpr (CG)
      for (int i = 0; i < 32; ++i) a = fmaf(__ldg(w + 48 + i), rec[C_CFEAT + i], a);
    for (int i = 0; i < 15; ++i) a = fmaf(__ldg(w + NC - 15 + i), so[1 + i], a);
    c1[j] = fmaxf(a, 0.f);
  }
  float o3[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) a = fmaf(__ldg(Q.w_col1 + k * 32 + i), c1[i], a);
    o3[k] = a;
  }
  *reinterpret_cast<float4*>(Q.raw + (size_t)p * 4) = make_float4(o3[0], o3[1], o3[2], so[0]);
}

__global__ void __launch_bounds__(128) k_query(const QueryParams Q) { query_points<false>(Q); }
__global__ void __launch_bounds__(128) k_query_c(const QueryParamsC Q) { query_points<true>(Q); }

static int fill_grid(GridDev& g, const XrdHashGrid* h) {
  if (h->n_levels < 1 || h->n_levels > kL) return XRD_E_SHAPE;
  g.n_levels = h->n_levels;
  for (int l = 0; l < kL; ++l) {
    g.scale[l] = h->scale[l]; g.res[l] = h->resolution[l]; g.size[l] = h->size[l] ? h->size[l] : 1;
    g.offset[l] = h->offset[l]; g.hashed[l] = h->hashed[l];
    g.magic[l] = (uint32_t)(0x100000000ull / g.size[l]);
  }
  for (int d = 0; d < 3; ++d) {
    g.bmin[d] = h->bbox_min[d]; g.bmax[d] = h->bbox_max[d];
    g.binv[d] = 1.0 / (h->bbox_max[d] - h->bbox_min[d]);
  }
  return XRD_OK;
}

// -------------------------------------------------------------- importance ---
// Hierarchical sampling between the coarse and the fine pass (joint_encoding.py:301-315), one
// warp per ray: sample_pdf (sample_pdf.cuh) on the coarse pass's weights (composite_weights on
// its raw sdf and z_vals, divided by their sum), z_fine = sort(z_vals ++ z_samples), the spread
// z_std of the samples and the fine pass's counts n_fs, n_sdf, n_valid over z_fine.
struct ImportanceParams {
  int R, S, N, det;
  float trunc, depth_trunc;
  const float *z_vals, *raw, *target_d, *u, *lin_u;
  uint64_t seed;
  const uint64_t* seed_dev;
  float *z_fine, *z_samples, *z_std;
  int* counts;
};
constexpr int kImpWarps = 4;
// shared floats per warp: sigma / pdf, weights, cdf, bin midpoints (S each), merged values (S + N)
__host__ __device__ constexpr int imp_floats(int S, int N) { return 4 * S + S + N; }

__global__ void __launch_bounds__(kImpWarps * 32) k_importance(ImportanceParams p) {
  extern __shared__ float ism[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * kImpWarps + warp;
  const int S = p.S, N = p.N, T = S + N;
  float* pdf = ism + (size_t)warp * imp_floats(S, N);
  float* wu = pdf + S;
  float* cdf = wu + S;
  float* mid = cdf + S;
  float* zall = mid + S;
  int c_fs = 0, c_sdf = 0, c_valid = 0;
  if (r < p.R) {  // warp-uniform
    const float* zr = p.z_vals + (size_t)r * S;
    // (COLOURS = false: raw is only read)
    const float W = composite_weights<4, 0, false>(const_cast<float*>(p.raw) + (size_t)r * S * 4,
                                                   zr, S, p.trunc, pdf, wu, lane);
    __syncwarp();  // the weights other lanes wrote in composite_weights are read below
    pdf_cdf([&](int j) { return wu[j] / W; }, zr, S, pdf, cdf, mid, zall, lane);
    const PdfDraw draw{p.u, p.lin_u, p.det, p.seed_dev ? *p.seed_dev : p.seed};
    invert_cdf(draw, r, S, N, cdf, mid, zall, p.z_samples ? p.z_samples + (size_t)r * N : nullptr,
               lane);
    rank_merge(zall, T, p.z_fine + (size_t)r * T, lane);
    if (p.counts) {
      const float d = p.target_d[r];
      for (int e = lane; e < T; e += 32) count_sample(zall[e], d, p.trunc, c_fs, c_sdf);
      if (lane == 0) c_valid = (d > 0.f && d < p.depth_trunc);
    }
    if (p.z_std) {  // std(z_samples, unbiased=False), two passes in float64
      double zsum = 0.0;
      for (int j = lane; j < N; j += 32) zsum += (double)zall[S + j];
      const double mean = warp_sum_d(zsum) / N;
      double v = 0.0;
      for (int j = lane; j < N; j += 32) {
        const double dz = (double)zall[S + j] - mean;
        v += dz * dz;
      }
      v = warp_sum_d(v);
      if (lane == 0) p.z_std[r] = (float)sqrt(v / N);
    }
  }
  if (p.counts) add_counts(p.counts, c_fs, c_sdf, c_valid, lane);
}

// the corner-pair scatter adds to the table gradient in 16-byte chunks
static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace coslam
}  // namespace xrd

using namespace xrd;
using namespace xrd::coslam;

// A 256-byte header that one memset clears: counts int[4] at +0, loss_acc double[4] at +64 and the
// grouped kernel's work queue at +128.  Then z_vals, R*S floats.
struct StepWs : Carver {
  StepWs(void* base, int n_rays, int n_samples)
      : Carver(base), hdr(take<char>(256)), z(take<float>((size_t)n_rays * n_samples)) {}
  char* hdr;
  float* z;
};

extern "C" size_t xrd_coslam_workspace_bytes(int n_rays, int n_samples) {
  return StepWs(nullptr, n_rays, n_samples).bytes();
}

static int pick_rays_per_tile(int S, int requested) {
  if (requested > 0) return requested;
  // largest NR with NR*S <= 224 -> for S=43: 5 rays, 215 points, 224 threads
  int nr = 224 / S;
  return nr < 1 ? 1 : nr;  // S in (224, 256]: one ray per 256-thread tile
}

template <bool BWD, bool PREC3, bool BPREC3>
struct TileKernel {
  static constexpr auto fn = &k_fused<BWD, PREC3, BPREC3, BWD ? 6 : 1>;
};
template <bool BWD, bool PREC3, bool BPREC3>
struct TileKernelC {
  static constexpr auto fn = &k_fused_c<BWD, PREC3, BPREC3, BWD ? 8 : 1>;
};
template <bool BWD, bool PREC3, bool BPREC3>
struct GroupedKernel {
  static constexpr auto fn = &k_fused_g<BWD, PREC3, BPREC3>;
};

// The instantiation of fused kernel K for a pass.  cfg.precision: 0 = 3xTF32 everywhere, 1 =
// 3xTF32 forward + TF32 backward, 2 = TF32 everywhere; NULL for a gradient pass in another mode.
template <template <bool, bool, bool> class K>
static decltype(K<false, false, false>::fn) fused_kernel(bool grads, int precision) {
  if (!grads) return precision <= 1 ? K<false, true, false>::fn : K<false, false, false>::fn;
  switch (precision) {
    case 0: return K<true, true, true>::fn;
    case 1: return K<true, true, false>::fn;
    case 2: return K<true, false, false>::fn;
    default: return nullptr;
  }
}

// Launches a fused kernel with smem bytes of dynamic shared memory on min(ctas, SMs x resident
// CTAs per SM) persistent CTAs.  XRD_E_SHAPE: no instantiation, or no CTA fits on an SM.
template <typename... A>
static int launch_fused(void (*kernel)(A...), int ctas, int threads, size_t smem,
                        cudaStream_t stream, A... args) {
  if (!kernel) return XRD_E_SHAPE;
  XRD_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  XRD_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem));
  if (occ < 1) return XRD_E_SHAPE;
  const int max_ctas = num_sms() * occ;
  {
    KernelTimer kt(stream);
    kernel<<<ctas < max_ctas ? ctas : max_ctas, threads, smem, stream>>>(args...);
  }
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_coslam_step(const XrdRays* rays, const XrdHashGrid* grid,
                               const XrdCoslamMlp* mlp, const XrdCoslamCfg* cfg,
                               const float* noise, XrdCoslamOut* out, XrdCoslamGrads* grads,
                               void* workspace, size_t workspace_bytes, void* stream_) {
  if (!rays || !grid || !mlp || !cfg || !out || !workspace) return XRD_E_NULL;
  if (!rays->rays_o || !rays->rays_d || !grid->table || !mlp->w_sdf0 || !mlp->w_sdf1 ||
      !mlp->w_col0 || !mlp->w_col1)
    return XRD_E_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int R = rays->n_rays, S = cfg->n_samples;
  if (R <= 0) return XRD_OK;
  if (S < 2 || S > 256) return XRD_E_SHAPE;
  const bool has_depth = rays->target_d != nullptr;
  // a fine pass (phase 2 on the z_vals of xrd_coslam_importance) marches n_importance more
  if (cfg->n_importance < 0) return XRD_E_SHAPE;
  const int n_fine = cfg->phase == 2 ? cfg->n_importance : 0;
  if (has_depth && S != cfg->n_sample_d + cfg->n_range_d + n_fine) return XRD_E_SHAPE;
  if (has_depth && (!cfg->lin_uniform || !cfg->lin_range || !cfg->lin_nodepth)) return XRD_E_NULL;
  if (!has_depth && !cfg->lin_full) return XRD_E_NULL;
  if (grads && (!has_depth || !rays->target_s || !out->losses)) return XRD_E_NULL;
  const XrdHashGrid* grid_c = mlp->grid_color;  // NULL: one grid (ColorSDFNet_v2)
  if (grid_c && !grid_c->table) return XRD_E_NULL;
  if (grads) {
    // map gradients are all-or-nothing; d_table == NULL selects the pose-only (tracking) pass
    const int n_map = (grads->d_table != nullptr) + (grads->d_w_sdf0 != nullptr) +
                      (grads->d_w_sdf1 != nullptr) + (grads->d_w_col0 != nullptr) +
                      (grads->d_w_col1 != nullptr) +
                      (grid_c ? (grads->d_table_color != nullptr) : 0);
    if (n_map != 0 && n_map != (grid_c ? 6 : 5)) return XRD_E_NULL;
    if (n_map == 0 && !grads->d_rays_o && !grads->d_rays_d) return XRD_E_NULL;
    if (grads->d_table && !aligned16(grads->d_table)) return XRD_E_SHAPE;
    if (grid_c && grads->d_table_color && !aligned16(grads->d_table_color)) return XRD_E_SHAPE;
  }
  const StepWs L(workspace, R, S);
  if (int st = L.check(workspace_bytes)) return st;

  int* counts = reinterpret_cast<int*>(L.hdr);  // n_fs, n_sdf, n_valid
  double* loss_acc = reinterpret_cast<double*>(L.hdr + 64);
  float* z_vals = out->z_vals ? out->z_vals : L.z;
  const int phase = cfg->phase;  // 0: sample+render, 1: sample only, 2: render only
  if (phase < 0 || phase > 2) return XRD_E_SHAPE;
  if (phase != 0 && !out->z_vals) return XRD_E_NULL;
  if (phase == 1 && !cfg->counts_out) return XRD_E_NULL;
  XRD_CUDA_TRY(cudaMemsetAsync(L.hdr, 0, 256, stream));
  if (phase == 1) {
    counts = cfg->counts_out;
    XRD_CUDA_TRY(cudaMemsetAsync(counts, 0, 4 * sizeof(int), stream));
  }
  SampleParams sp;
  sp.R = R; sp.S = S; sp.n_a = cfg->n_sample_d; sp.n_b = cfg->n_range_d;
  sp.perturb = cfg->perturb; sp.has_depth = has_depth;
  sp.target_d = rays->target_d; sp.lin_uniform = cfg->lin_uniform; sp.lin_range = cfg->lin_range;
  sp.lin_nodepth = cfg->lin_nodepth; sp.lin_full = cfg->lin_full; sp.noise = noise;
  sp.trunc = cfg->trunc; sp.depth_trunc = cfg->depth_trunc; sp.seed = cfg->seed;
  sp.seed_dev = cfg->seed_dev;
  sp.z_vals = z_vals; sp.counts = counts;
  if (phase != 2) {
    k_sample<<<(R + 3) / 4, 128, 0, stream>>>(sp);
    XRD_LAUNCH_CHECK();
  }
  if (phase == 1) return XRD_OK;

  ParamsC P;  // k_fused and k_fused_g take its Params part
  int st = fill_grid(P.g, grid);
  if (st != XRD_OK) return st;
  P.R = R; P.S = S;
  P.Rg = cfg->n_rays_global > 0 ? cfg->n_rays_global : R;
  P.rays_o = rays->rays_o; P.rays_d = rays->rays_d; P.target_s = rays->target_s; P.target_d = rays->target_d;
  P.z_vals = z_vals; P.table = grid->table;
  P.w_sdf0 = mlp->w_sdf0; P.w_sdf1 = mlp->w_sdf1; P.w_col0 = mlp->w_col0; P.w_col1 = mlp->w_col1;
  P.trunc = cfg->trunc; P.depth_trunc = cfg->depth_trunc;
  P.w_rgb = cfg->w_rgb; P.w_depth = cfg->w_depth; P.w_sdf = cfg->w_sdf; P.w_fs = cfg->w_fs;
  P.rgb = out->rgb; P.depth = out->depth; P.disp = out->disp; P.acc = out->acc;
  P.depth_var = out->depth_var; P.raw = out->raw;
  P.counts = cfg->counts_global ? cfg->counts_global : counts; P.loss_acc = loss_acc;
  for (int i = 0; i < 4; ++i) P.ls[i] = grads ? grads->loss_scale[i] : 0.f;
  if (grads) {
    P.d_table = grads->d_table; P.d_w_sdf0 = grads->d_w_sdf0; P.d_w_sdf1 = grads->d_w_sdf1;
    P.d_w_col0 = grads->d_w_col0; P.d_w_col1 = grads->d_w_col1;
    P.d_rays_o = grads->d_rays_o; P.d_rays_d = grads->d_rays_d;
  } else {
    P.d_table = P.d_w_sdf0 = P.d_w_sdf1 = P.d_w_col0 = P.d_w_col1 = P.d_rays_o = P.d_rays_d = nullptr;
  }
  P.table_c = nullptr;
  P.d_table_c = nullptr;
  if (grid_c) {
    st = fill_grid(P.gc, grid_c);
    if (st != XRD_OK) return st;
    P.table_c = grid_c->table;
    P.d_table_c = grads ? grads->d_table_color : nullptr;
  }
  const int sms = num_sms();
  // Kernel choice (rays_per_tile: 0 = automatic, -1 = tile kernel, -2 = grouped kernel, > 0 = tile
  // kernel with that many rays per tile).  Automatic: the grouped kernel runs the gradient pass
  // once every group has >= 1 unit in flight after the first wave; the tile kernel runs small
  // batches (tracking) and forward-only rendering.  On H100 (400 W) the grouped kernel takes
  // 0.433 ms of the benchmark's 4096-ray mapping step.  On scripts/quick_time_coslam.py's
  // random rays (mode 1) the two are close: tile / grouped fwd+bwd R = 1024: 214 / 195 us,
  // 4096: 462 / 468, 16384: 1470 / 1520, 65536: 5463 / 5818 us; the rule is unchanged.
  // A colour-grid pass runs on the tile kernel: the grouped kernel's three groups of 96 records
  // would need 32 more floats each, which with its weight-gradient buffer outgrows the 227 KB a
  // CTA may opt in to.
  if (grid_c && cfg->rays_per_tile == -2) return XRD_E_SHAPE;
  bool grouped = false;
  if (S <= GP && !grid_c) {
    const int units = (R + GP / S - 1) / (GP / S);
    grouped = cfg->rays_per_tile == -2 || (cfg->rays_per_tile == 0 && grads && units >= 4 * sms);
  }
  if (grouped) {
    // grouped persistent kernel (k_fused_g): units of NR rays pulled from a queue
    P.NR = GP / S;
    P.n_tiles = (R + P.NR - 1) / P.NR;
    int* queue = reinterpret_cast<int*>(L.hdr + 128);  // zeroed above
    // weights + NGROUPS x GP records + one z value per slot: 180 352 B, plus 18 432 B of
    // weight-gradient buffer when map gradients are on.  Four groups would fit (231 424 B) but
    // need <= 80 registers per thread and spill more; with three, what the 196 KB configuration
    // leaves of the SM's 256 KB serves as L1 for the gathers (1.25x the step rate on H100).
    const size_t smem_g = P.d_table ? G_SMEM_DW : G_SMEM;
    const auto kernel = fused_kernel<GroupedKernel>(grads != nullptr, cfg->precision);
    if (!kernel) return XRD_E_SHAPE;
    int dev = 0, smem_optin = 0;
    cudaFuncAttributes fa;
    XRD_CUDA_TRY(cudaGetDevice(&dev));
    XRD_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    XRD_CUDA_TRY(cudaFuncGetAttributes(&fa, kernel));
    if (smem_g + fa.sharedSizeBytes > (size_t)smem_optin) return XRD_E_SHAPE;
    st = launch_fused(kernel, (P.n_tiles + NGROUPS - 1) / NGROUPS, GT * NGROUPS, smem_g, stream,
                      static_cast<const Params&>(P), queue);
  } else {
    // tile kernel (k_fused): rays_per_tile > 0 selects its tile size, < 0 its default
    const int NR = pick_rays_per_tile(S, cfg->rays_per_tile);
    if (NR < 1 || NR * S > 256) return XRD_E_SHAPE;
    int threads = (NR * S + 31) / 32 * 32;
    if (grads && threads < 224) threads = 224;  // 7+ warps own the 42 weight-gradient tiles (6 each)
    P.NR = NR;
    P.n_tiles = (R + NR - 1) / NR;
    if (!grid_c) {
      if (grads && (DW_TILES + threads / 32 - 1) / (threads / 32) != 6) return XRD_E_SHAPE;
      // weights + (threads + 8) records + per point z and xn
      const size_t smem = sizeof(float) * ((size_t)SW_TOTAL + (size_t)(threads + 8) * REC + 6 * (size_t)NR * S);
      st = launch_fused(fused_kernel<TileKernel>(grads != nullptr, cfg->precision), P.n_tiles,
                        threads, smem, stream, static_cast<const Params&>(P));
    } else {
      // 50 weight-gradient tiles: 8 slots per warp cover them from 7 warps on
      if (grads && (Wts<true>::DW + threads / 32 - 1) / (threads / 32) > 8) return XRD_E_SHAPE;
      // gradient pass, 224 threads (S = 43): 219 304 B of the 227 KB opt-in (NR * S above 224
      // does not fit); forward only, compact record: 177 792 B at 256 threads
      const size_t smem = sizeof(float) * ((size_t)Wts<true>::TOTAL +
                                           (size_t)(threads + 8) * (grads ? CREC : FREC) +
                                           6 * (size_t)NR * S);
      int dev = 0, smem_optin = 0;
      XRD_CUDA_TRY(cudaGetDevice(&dev));
      XRD_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
      if (smem + 2 * kL * sizeof(Lv) > (size_t)smem_optin) return XRD_E_SHAPE;
      st = launch_fused(fused_kernel<TileKernelC>(grads != nullptr, cfg->precision), P.n_tiles,
                        threads, smem, stream, P);
    }
  }
  if (st != XRD_OK || !grads) return st;
  FinalizeParams fp{loss_acc, P.counts, out->losses, P.Rg, S, cfg->w_rgb, cfg->w_depth, cfg->w_sdf, cfg->w_fs};
  k_finalize<<<1, 32, 0, stream>>>(fp);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_coslam_importance(const XrdCoslamImportance* q, void* stream_) {
  if (!q || !q->z_vals || !q->raw || !q->z_fine) return XRD_E_NULL;
  const int R = q->n_rays, S = q->n_samples, N = q->n_importance;
  // the fine pass marches S + N samples per ray: at most 256 (xrd_coslam_step)
  if (R < 0 || S < 3 || N < 1 || S + N > 256) return XRD_E_SHAPE;
  if (!q->u && q->det && !q->lin_u) return XRD_E_NULL;
  if (q->counts_out && !q->target_d) return XRD_E_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (q->counts_out) XRD_CUDA_TRY(cudaMemsetAsync(q->counts_out, 0, 4 * sizeof(int), stream));
  if (R == 0) return XRD_OK;
  ImportanceParams p;
  p.R = R; p.S = S; p.N = N; p.det = q->det;
  p.trunc = q->trunc; p.depth_trunc = q->depth_trunc;
  p.z_vals = q->z_vals; p.raw = q->raw; p.target_d = q->target_d; p.u = q->u; p.lin_u = q->lin_u;
  p.seed = q->seed; p.seed_dev = q->seed_dev;
  p.z_fine = q->z_fine; p.z_samples = q->z_samples; p.z_std = q->z_std; p.counts = q->counts_out;
  const size_t smem = sizeof(float) * kImpWarps * (size_t)imp_floats(S, N);  // <= 20 KB
  k_importance<<<(R + kImpWarps - 1) / kImpWarps, kImpWarps * 32, smem, stream>>>(p);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

// xrd_debug_smooth_box_cap: an upper limit on the box capacity, per calling thread (< 0: none)
thread_local int g_smooth_box_cap = -1;

// the loss accumulator and the CTA counter of k_smooth_bwd
struct SmoothWs : Carver {
  explicit SmoothWs(void* base) : Carver(base) {}
  SmoothHdr* hdr = take_last<SmoothHdr>(1);
};

extern "C" size_t xrd_coslam_smoothness_workspace_bytes(int sample_points) {
  (void)sample_points;
  return SmoothWs(nullptr).bytes();
}

static int smoothness_impl(const XrdHashGrid* grid, int sample_points, double voxel_size,
                           double margin, float weight, const float* smooth_rand, bool rand_on_device,
                           float* loss, float* d_table, float grad_scale,
                           void* workspace, size_t workspace_bytes, void* stream_) {
  if (!grid || !grid->table || !smooth_rand || !loss || !workspace) return XRD_E_NULL;
  if (sample_points < 3 || sample_points - 1 > kSmoothMaxN) return XRD_E_SHAPE;
  if (d_table && !aligned16(d_table)) return XRD_E_SHAPE;
  const SmoothWs L(workspace);
  if (int st = L.check(workspace_bytes)) return st;
  cudaStream_t stream = (cudaStream_t)stream_;
  SmoothParams p;
  int st = fill_grid(p.g, grid);
  if (st != XRD_OK) return st;
  p.table = grid->table;
  p.n = sample_points - 1;
  // joint_encoding.py:171-181 -- float64 throughout (bounding_box is a float64 tensor); the
  // python floats voxel_size/margin enter as doubles, the two torch.rand draws as float32
  p.voxel = voxel_size;
  const double grid_size = (double)(sample_points - 1) * voxel_size;
  for (int d = 0; d < 3; ++d) {
    double offset_max = grid->bbox_max[d] - grid->bbox_min[d] - grid_size - 2.0 * margin;
    p.offmax[d] = offset_max;
    p.off[d] = rand_on_device ? 0.0 : (double)smooth_rand[d] * offset_max + margin;
    p.rnd[d] = rand_on_device ? 0.0 : (double)smooth_rand[3 + d];
  }
  p.margin = margin;
  p.rand_dev = rand_on_device ? smooth_rand : nullptr;
  p.hdr = L.hdr;
  p.loss = loss;
  p.d_table = d_table;
  const double sp3 = (double)sample_points * sample_points * sample_points;
  p.coef = (float)((double)grad_scale * (double)weight / sp3);
  p.loss_scale = (float)((double)weight / sp3);
  // the window and the point gradients, then as large a box as the rest of the SM's shared
  // memory holds (up to kSmoothBox entries)
  int dev = 0, smem_optin = 0;
  cudaFuncAttributes fa;
  XRD_CUDA_TRY(cudaGetDevice(&dev));
  XRD_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  XRD_CUDA_TRY(cudaFuncGetAttributes(&fa, k_smooth_bwd));
  const size_t win = 5 * sizeof(float2) * (size_t)p.n * p.n;
  const long long room = ((long long)smem_optin - (long long)fa.sharedSizeBytes - (long long)win) /
                         (2 * (long long)sizeof(float2));
  if (room < 0) return XRD_E_SHAPE;
  p.box_cap = (int)(room < kSmoothBox ? room : kSmoothBox);
  if (g_smooth_box_cap >= 0 && g_smooth_box_cap < p.box_cap) p.box_cap = g_smooth_box_cap;
  const size_t smem = win + 2 * sizeof(float2) * (size_t)p.box_cap;
  XRD_CUDA_TRY(cudaFuncSetAttribute(k_smooth_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem));
  // the caller's workspace arrives uninitialised: zero the 16-byte header every call
  XRD_CUDA_TRY(cudaMemsetAsync(L.hdr, 0, sizeof(SmoothHdr), stream));
  const dim3 blocks((p.n + kSmoothPlanes - 1) / kSmoothPlanes, p.g.n_levels);
  k_smooth_bwd<<<blocks, kSmoothThreads, smem, stream>>>(p);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_coslam_smoothness(const XrdHashGrid* grid, int sample_points, double voxel_size,
                                     double margin, float weight, const float* smooth_rand,
                                     float* loss, float* d_table, float grad_scale,
                                     void* workspace, size_t workspace_bytes, void* stream_) {
  return smoothness_impl(grid, sample_points, voxel_size, margin, weight, smooth_rand, false, loss,
                         d_table, grad_scale, workspace, workspace_bytes, stream_);
}

extern "C" int xrd_coslam_smoothness_dev(const XrdHashGrid* grid, int sample_points, double voxel_size,
                                         double margin, float weight, const float* smooth_rand,
                                         float* loss, float* d_table, float grad_scale,
                                         void* workspace, size_t workspace_bytes, void* stream_) {
  return smoothness_impl(grid, sample_points, voxel_size, margin, weight, smooth_rand, true, loss,
                         d_table, grad_scale, workspace, workspace_bytes, stream_);
}

extern "C" int xrd_debug_smooth_box_cap(int cap) {
  const int prev = g_smooth_box_cap;
  g_smooth_box_cap = cap < 0 ? -1 : cap;
  return prev;
}

extern "C" int xrd_coslam_query(const XrdHashGrid* grid, const XrdCoslamMlp* mlp, const float* pts,
                                int n_points, int normalised, float* raw, float* geo, float* feat,
                                void* stream_) {
  if (!grid || !grid->table || !pts) return XRD_E_NULL;
  if ((raw || geo) && (!mlp || !mlp->w_sdf0 || !mlp->w_sdf1)) return XRD_E_NULL;
  if (raw && (!mlp->w_col0 || !mlp->w_col1)) return XRD_E_NULL;
  const XrdHashGrid* grid_c = mlp ? mlp->grid_color : nullptr;
  if (grid_c && !grid_c->table) return XRD_E_NULL;
  if (n_points <= 0) return XRD_OK;
  QueryParamsC Q;  // k_query takes its QueryParams part
  int st = fill_grid(Q.g, grid);
  if (st != XRD_OK) return st;
  Q.table = grid->table;
  Q.w_sdf0 = mlp ? mlp->w_sdf0 : nullptr; Q.w_sdf1 = mlp ? mlp->w_sdf1 : nullptr;
  Q.w_col0 = mlp ? mlp->w_col0 : nullptr; Q.w_col1 = mlp ? mlp->w_col1 : nullptr;
  Q.pts = pts; Q.P = n_points; Q.normalised = normalised; Q.raw = raw; Q.geo = geo; Q.feat = feat;
  Q.table_c = nullptr;
  if (grid_c) {
    st = fill_grid(Q.gc, grid_c);
    if (st != XRD_OK) return st;
    Q.table_c = grid_c->table;
  }
  const size_t smem = 128 * (grid_c ? CREC : REC) * sizeof(float);
  if (grid_c) {
    XRD_CUDA_TRY(cudaFuncSetAttribute(k_query_c, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_query_c<<<(n_points + 127) / 128, 128, smem, (cudaStream_t)stream_>>>(Q);
  } else {
    XRD_CUDA_TRY(cudaFuncSetAttribute(k_query, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_query<<<(n_points + 127) / 128, 128, smem, (cudaStream_t)stream_>>>(Q);
  }
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}

extern "C" int xrd_hashgrid_encode(const XrdHashGrid* grid, const float* x, int n_points,
                                   float* feat, uint32_t* idx, void* stream_) {
  if (!grid || !grid->table || !x) return XRD_E_NULL;
  if (n_points <= 0) return XRD_OK;
  GridDev g;
  int st = fill_grid(g, grid);
  if (st != XRD_OK) return st;
  const long long total = (long long)n_points * kL;
  k_encode<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(g, grid->table, x, n_points, feat, idx);
  XRD_LAUNCH_CHECK();
  return XRD_OK;
}
