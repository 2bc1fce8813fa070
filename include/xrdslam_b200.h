/*
 * xrdslam_b200 -- C-ABI of the H100-native render-and-optimise hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point is
 * `extern "C"`, takes plain pointers / sizes / POD structs, never allocates,
 * never frees, never synchronises the stream: one call = an asynchronous enqueue
 * of sm_90a kernels on `stream` (a cudaStream_t passed as void*).  All buffers,
 * including the workspace, are owned by the caller (torch on the Python side).
 * Return value: XRD_OK (0) or a negative XrdStatus.  No exceptions, no exit().
 *
 * What each entry point replaces in the reference (paths relative to the
 * xrdslam repository, commit f0366f20):
 *
 *   xrd_coslam_step        slam/models/joint_encoding.py:158-163  get_outputs
 *                          -> render_rays :250-344, run_network :483-507,
 *                          query_color_sdf :463-481 (tcnn HashGrid + OneBlob via
 *                          slam/model_components/encodings_coslam.py:39-75,
 *                          decoders slam/model_components/decoder_coslam.py:139-163),
 *                          sdf2weights :346-374, raw2outputs :376-406,
 *                          get_loss_dict :94-147 (+ utils.py:100-186) and the
 *                          autograd backward of all of it (loss.backward(),
 *                          slam/algorithms/base_algorithm.py:266).
 *   xrd_coslam_smoothness  slam/models/joint_encoding.py:165-197 smoothness
 *                          (forward + gradient w.r.t. the hash table).
 *   xrd_hashgrid_layout    tcnn GridEncodingTemplated ctor (level offsets), the
 *                          config built at encodings_coslam.py:39-53.
 *   xrd_linspace_f32       torch.linspace as used at joint_encoding.py:264-279.
 *
 * (NICE-SLAM / Vox-Fusion / Point-SLAM entry points are declared further down.)
 */
#ifndef XRDSLAM_B200_H_
#define XRDSLAM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XRD_ABI_VERSION 1
#define XRD_MAX_LEVELS 16

typedef enum {
  XRD_OK = 0,
  XRD_E_SHAPE = -1,     /* inconsistent sizes / unsupported configuration   */
  XRD_E_ARCH = -2,      /* device is not sm_90                               */
  XRD_E_WORKSPACE = -3, /* workspace too small                               */
  XRD_E_NOHIT = -4,     /* Vox-Fusion: no ray hit any voxel (reference: None) */
  XRD_E_CUDA = -5,      /* a CUDA runtime call failed (see xrd_last_cuda_error) */
  XRD_E_NULL = -6       /* a required pointer is NULL                        */
} XrdStatus;

int xrd_abi_version(void);
/* cudaError_t of the last failing runtime call on this thread (0 if none). */
int xrd_last_cuda_error(void);
/* 0 if device `dev` is compute capability 10.x, XRD_E_ARCH otherwise. */
int xrd_check_device(int dev);

/* Measurement hook (bench.py roofline): when both events are non-NULL the NEXT
 * dominant-kernel launch made from this thread (k_fused of xrd_coslam_step, the
 * fused render kernels of the other representations) is bracketed by
 * cudaEventRecord(start)/(stop) on the launching stream.  Pass NULL, NULL to
 * clear.  The events are cudaEvent_t handles owned by the caller. */
int xrd_debug_kernel_events(void* start_event, void* stop_event);

/* ---- shared ------------------------------------------------------------ */

/* A batch of rays.  All pointers are DEVICE pointers, fp32, contiguous. */
typedef struct {
  int n_rays;
  const float* rays_o;   /* [R,3] */
  const float* rays_d;   /* [R,3] */
  const float* target_s; /* [R,3] colour target, may be NULL (render only)   */
  const float* target_d; /* [R]   depth target,  may be NULL                 */
} XrdRays;

/* torch.linspace(start, end, steps) for float32 by ATen's scalar formula (host
 * function, writes `steps` floats to host memory `out`).  ATen's vectorised CPU
 * path differs in the last bit for some elements depending on the host's SIMD
 * width; callers that need the reference's exact z samples pass tables made by
 * torch.linspace on the same host (the Python plugin does). */
int xrd_linspace_f32(float start, float end, int steps, float* out);

/* ---- shared front-end / optimiser (SURVEY rows A2, A7, B3; "next" row f1) ---------- */

/* World-frame rays from camera-frame directions and a per-ray pose row:
 *   rays_d[r] = sum_j dirs_cam[r][j] * poses[id][:3, j],  rays_o[r] = poses[id][:3, 3]
 * replaces slam/common/common.py:39-53 (get_rays_from_uv) and the per-ray pose gather of
 * slam/algorithms/coslam.py:208-216.  poses: DEVICE [n_poses,4,4] row-major c2w; pose_ids:
 * DEVICE [R] int64 or NULL (all rays use pose 0); negative ids index from the end (python). */
int xrd_rays_from_poses(int n_rays, const float* dirs_cam, const int64_t* pose_ids,
                        const float* poses, int n_poses, float* rays_o, float* rays_d,
                        void* stream);

/* Backward of the above: d_poses [n_poses,4,4] (zeroed inside, bottom row stays 0)
 *   d_poses[id][:3,:3] += outer(d_rays_d[r], dirs_cam[r]),  d_poses[id][:3,3] += d_rays_o[r]
 * (what torch's index_put(accumulate=True) backward of `poses_all[ids]` computes). */
int xrd_rays_pose_grads(int n_rays, const float* dirs_cam, const int64_t* pose_ids, int n_poses,
                        const float* d_rays_o, const float* d_rays_d, float* d_poses,
                        void* stream);

/* Pixel sampling for a window of frames in one launch: gathers depth / colour of the chosen
 * pixels of device-resident frames and builds the camera-frame directions
 *   dirs = [(i - cx) / fx, -(j - cy) / fy, -1],  i = idx % (W1 - W0) + W0,  j = idx / (W1 - W0) + H0
 * (slam/common/common.py:56-71 select_uv, :109-122 get_sample_uv, :45-47; the reference
 * re-uploads both full images for every frame of every iteration).  indices: DEVICE
 * [n_frames * n_per_frame] int64 into the cropped region (row-major), frame-major; the draw
 * itself (torch.randint, with replacement, Q7) stays with the caller.  depth_imgs / rgb_imgs:
 * HOST arrays of n_frames DEVICE pointers ([H,W] and [H,W,3] fp32).  Outputs are frame-major;
 * pose_ids[q] = frame index (feeds xrd_rays_from_poses); ij: optional [n,2] (column, row). */
typedef struct {
  int n_frames;    /* <= 32 */
  int n_per_frame;
  int H, W;        /* image size */
  int H0, H1, W0, W1; /* sampled region (Hedge / Wedge crop) */
  float fx, fy, cx, cy;
} XrdPixelSampleCfg;

int xrd_sample_pixels(const XrdPixelSampleCfg* cfg, const float* const* depth_imgs,
                      const float* const* rgb_imgs, const int64_t* indices, float* dirs,
                      float* depth, float* rgb, int64_t* pose_ids, int64_t* ij, void* stream);

/* c2w [n,4,4] from axis-angle `rot` [n,3] and translation `trans` [n,3] (all DEVICE):
 * slam/utils/opt_pose.py:51-55,77-95 (OptimizablePose.matrix / Rodrigues). */
int xrd_pose_matrices(int n_poses, const float* rot, const float* trans, float* c2w, void* stream);

/* Backward of the above (what torch autograd computes through opt_pose.py): d_rot / d_trans
 * [n,3] are ACCUMULATED into (Co-SLAM steps its mapping poses every 5th iteration on the summed
 * gradients, SURVEY Q11).  fixed: DEVICE [n] or NULL; rows with fixed != 0 receive nothing
 * (the first frame of the window, coslam.py:181-182 / base_algorithm.py:196-199). */
int xrd_pose_matrices_grads(int n_poses, const float* rot, const float* d_c2w,
                            const uint8_t* fixed, float* d_rot, float* d_trans, void* stream);

/* One tensor of a multi-tensor Adam step (torch.optim.Adam, amsgrad=False); all DEVICE fp32.
 * bias_correction{1,2} = 1 - beta{1,2}^step with step counted from 1 (host, double -> float). */
#define XRD_ADAM_MAX_TENSORS 24
typedef struct {
  float* param; float* grad; float* exp_avg; float* exp_avg_sq;
  long long n;
  float lr, beta1, beta2, eps, weight_decay, bias_correction1, bias_correction2;
  /* optional row mask: element i is updated only if row_mask[i / row_len] != 0.  This is the
   * frustum feature selection of NICE-SLAM (slam/models/conv_onet.py:94-114,187-211: the
   * reference optimises a compacted copy val[mask] and scatters it back into the full grid
   * every iteration); rows = voxels of the channel-last grid, row_len = 32. */
  const uint8_t* row_mask;
  int row_len;
  /* optional DEVICE [3] = {lr, bias_correction1, bias_correction2} overriding the host values:
   * lets a captured CUDA graph replay the step with per-iteration scalars. */
  const float* dyn;
} XrdAdamTensor;

/* tensors: HOST array.  zero_grad != 0 also clears every grad (folds zero_grad_all,
 * slam/engine/optimizers.py:150-162, into the pass).  Replaces optimizer_step_all (:125-148)
 * for device-resident parameter groups. */
int xrd_adam_step(const XrdAdamTensor* tensors, int n_tensors, int zero_grad, void* stream);

/* ---- Co-SLAM ------------------------------------------------------------ */

/* Multi-resolution hash grid in tcnn's parameter layout: one flat fp32 array,
 * level-major, entry-major, feature-minor, 2 features per entry. */
typedef struct {
  int n_levels;                        /* <= XRD_MAX_LEVELS (Co-SLAM: 16)      */
  float scale[XRD_MAX_LEVELS];         /* grid_scale(level)                    */
  uint32_t resolution[XRD_MAX_LEVELS]; /* grid_resolution(scale)               */
  uint32_t size[XRD_MAX_LEVELS];       /* entries in level                     */
  uint32_t offset[XRD_MAX_LEVELS];     /* first entry of level                 */
  uint32_t hashed[XRD_MAX_LEVELS];     /* 1: coherent-prime hash, 0: dense     */
  uint32_t n_entries;                  /* sum(size)                            */
  double bbox_min[3];                  /* scene bound, float64 as the reference */
  double bbox_max[3];
  const float* table;                  /* DEVICE [n_entries*2]                 */
} XrdHashGrid;

/* Fill scale/resolution/size/offset/hashed/n_entries (host function). */
int xrd_hashgrid_layout(XrdHashGrid* g, int n_levels, int log2_hashmap_size,
                        int base_resolution, float per_level_scale);

/* ColorSDFNet_v2 weights, torch nn.Linear layout [out,in], no bias. DEVICE. */
typedef struct {
  const float* w_sdf0; /* [32,80]  in = hash32 ++ oneblob48                  */
  const float* w_sdf1; /* [16,32]  out = sdf ++ geo15                        */
  const float* w_col0; /* [32,63]  in = oneblob48 ++ geo15                   */
  const float* w_col1; /* [3,32]                                             */
} XrdCoslamMlp;

typedef struct {
  int n_samples;      /* S: samples per ray actually marched (43 with depth) */
  int n_sample_d;     /* 32 uniform samples in [near,far]                    */
  int n_range_d;      /* 11 depth-guided samples                             */
  int perturb;        /* stratified jitter on/off                            */
  float trunc;        /* training_trunc * sc_factor (0.1)                    */
  float depth_trunc;  /* cam_depth_trunc (100)                               */
  float w_rgb, w_depth, w_sdf, w_fs; /* loss weights 5, 0.1, 1000, 10        */
  /* DEVICE tables, normally produced with torch.linspace / xrd_linspace_f32: */
  const float* lin_uniform;  /* [n_sample_d]  linspace(near, far)             */
  const float* lin_range;    /* [n_range_d]   linspace(-range_d, range_d)     */
  const float* lin_nodepth;  /* [n_range_d]   linspace(near, far)             */
  const float* lin_full;     /* [n_samples]   used when target_d == NULL      */
  uint64_t seed;             /* Philox seed when noise == NULL                */
  int rays_per_tile;         /* 0 = automatic (grouped kernel for large gradient
                              * batches, tile kernel otherwise); -1 = tile kernel,
                              * -2 = grouped kernel, > 0 = tile kernel, rays/tile */
  int precision;             /* decoder GEMMs on the tensor cores:
                              * 0 = 3xTF32 everywhere (fp32-level accuracy),
                              * 1 = 3xTF32 forward (outputs/losses fp32-level),
                              *     plain TF32 backward (gradients ~1e-3 rel),
                              * 2 = plain TF32 everywhere                       */
  /* data-parallel mapping (loss normalisers are batch-global, SURVEY Q9):       */
  int phase;                 /* 0 = sample+render, 1 = sample only (z_vals and
                              * counts_out), 2 = render only (z_vals given)     */
  int n_rays_global;         /* rays of the all-rank batch; 0 = n_rays          */
  const int* counts_global;  /* DEVICE [3] n_fs, n_sdf, n_valid of the all-rank
                              * batch; NULL = this call's own counts            */
  int* counts_out;           /* DEVICE [4], written in phase 1                  */
  const uint64_t* seed_dev;  /* DEVICE scalar overriding `seed` (read by the kernel:
                              * a captured CUDA graph replays with a fresh seed)  */
} XrdCoslamCfg;

/* Per-ray / per-sample outputs (DEVICE, any may be NULL except losses when
 * grads are requested). */
typedef struct {
  float* rgb;       /* [R,3] */
  float* depth;     /* [R]   */
  float* disp;      /* [R]   */
  float* acc;       /* [R]   */
  float* depth_var; /* [R]   */
  float* z_vals;    /* [R,S] */
  float* raw;       /* [R,S,4] rgb logits ++ sdf */
  float* losses;    /* [4] rgb, depth, sdf, fs -- already multiplied by w_*  */
} XrdCoslamOut;

/* Gradients of (rgb+depth+sdf+fs) loss scaled by loss_scale[4] per term.
 * d_table and d_w_* are ACCUMULATED into (caller zeroes them: mapping-pose Adam
 * uses accum_step, Q11); d_rays_* are overwritten.  The five map gradients are
 * all-or-nothing: all NULL selects the pose-only pass used by tracking (no
 * scatter, no weight-gradient tiles).  d_table must be 16-byte aligned: two
 * x-adjacent trilinear corners that share a 16-byte chunk are added with one
 * vector reduction (XRD_E_SHAPE otherwise). */
typedef struct {
  float* d_table;  /* [n_entries*2] */
  float* d_w_sdf0; /* [32,80] */
  float* d_w_sdf1; /* [16,32] */
  float* d_w_col0; /* [32,63] */
  float* d_w_col1; /* [3,32]  */
  float* d_rays_o; /* [R,3] or NULL */
  float* d_rays_d; /* [R,3] or NULL */
  float loss_scale[4]; /* upstream d total / d term (normally 1,1,1,1) */
} XrdCoslamGrads;

size_t xrd_coslam_workspace_bytes(int n_rays, int n_samples);

/* One fused forward(+backward) pass.  noise: DEVICE [R,S] uniform(0,1) replacing
 * torch.rand(z_vals.shape) (joint_encoding.py:292) or NULL for in-kernel Philox.
 * grads == NULL -> forward only (render_img). */
int xrd_coslam_step(const XrdRays* rays, const XrdHashGrid* grid,
                    const XrdCoslamMlp* mlp, const XrdCoslamCfg* cfg,
                    const float* noise, XrdCoslamOut* out,
                    XrdCoslamGrads* grads, void* workspace,
                    size_t workspace_bytes, void* stream);

size_t xrd_coslam_smoothness_workspace_bytes(int sample_points);

/* Smoothness / TV regulariser on the hash features (joint_encoding.py:165-197).
 * smooth_rand: HOST [6] = torch.rand(3) ++ torch.rand((1,1,1,3)).  Writes
 * weight*loss to DEVICE loss[0]; if d_table != NULL accumulates
 * grad_scale*weight*dloss/dtable into it (16-byte aligned, as in XrdCoslamGrads). */
/* (xrd_coslam_smoothness_dev: the same with smooth_rand in DEVICE memory, read by the
 * kernels -- for CUDA-graph replay.) */
int xrd_coslam_smoothness(const XrdHashGrid* grid, int sample_points,
                          double voxel_size, double margin, float weight,
                          const float* smooth_rand, float* loss, float* d_table,
                          float grad_scale, void* workspace,
                          size_t workspace_bytes, void* stream);
int xrd_coslam_smoothness_dev(const XrdHashGrid* grid, int sample_points,
                          double voxel_size, double margin, float weight,
                          const float* smooth_rand, float* loss, float* d_table,
                          float grad_scale, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Point queries of the mesher path (slam/models/joint_encoding.py:408-481 query_fn /
 * color_func / query_sdf / query_color_sdf; slam/common/mesher.py:138-263 calls them on
 * marching-cubes lattice points): pts DEVICE [P,3], world coordinates (normalised = 0: the
 * kernel applies (p - bbox_min) / (bbox_max - bbox_min) in float64 like the reference) or
 * already normalised (1).  Any of raw [P,4] (rgb logits ++ sdf), geo [P,15], feat [P,32]
 * (hash features, query_sdf(embed=True)) may be NULL. */
int xrd_coslam_query(const XrdHashGrid* grid, const XrdCoslamMlp* mlp, const float* pts,
                     int n_points, int normalised, float* raw, float* geo, float* feat,
                     void* stream);

/* Hash-grid encoding only (used by the mesher path query_sdf(embed=True) and
 * by the index-parity tests): x DEVICE [P,3] normalised coords ->
 * feat [P,2*n_levels]; idx (optional) [P,n_levels,8] uint32 entry indices. */
int xrd_hashgrid_encode(const XrdHashGrid* grid, const float* x, int n_points,
                        float* feat, uint32_t* idx, void* stream);

/* ---- NICE-SLAM -------------------------------------------------------------
 *
 *   xrd_nice_step   slam/models/conv_onet.py:132-143 get_outputs -> render_batch_ray
 *                   :377-524 (bbox far plane, 32 uniform + 16 surface samples in float64,
 *                   sort), eval_points :339-375, NICE.forward
 *                   slam/model_components/decoder_nice.py:386-414 with the three MLP
 *                   decoders :207-234 (F.grid_sample trilerp :195-205, Gaussian Fourier
 *                   embedding :11-38), raw2outputs_nerf_color
 *                   slam/model_components/utils.py:189-244, get_loss_dict
 *                   conv_onet.py:145-185 (incl. the batch-global median of the tracking
 *                   mask) and autograd's backward.
 *
 * Feature grids are CHANNEL-LAST fp32 [Z][Y][X][32] (the reference holds [1,32,Z,Y,X];
 * one voxel = one 128-byte line here).  Decoder weights keep torch's [out,in] layout. */

typedef struct {
  const float* B;        /* [3][93]   Gaussian Fourier matrix (embedder._B)      */
  const float* pts_w[5]; /* [32][in]  in = 93, 32, 32, 125 (cat[embed, h]), 32     */
  const float* pts_b[5]; /* [32]                                                   */
  const float* fcc_w[5]; /* [32][c_dim]                                            */
  const float* fcc_b[5]; /* [32]                                                   */
  const float* out_w;    /* [n_out][32]                                            */
  const float* out_b;    /* [n_out]                                                */
  int c_dim;             /* 32 (middle, color) or 64 (fine: own grid ++ middle)    */
  int n_out;             /* 1 (occupancy) or 4 (colour decoder)                    */
} XrdNiceDecoder;

typedef struct {          /* same shapes as XrdNiceDecoder, ACCUMULATED into       */
  float* B;
  float* pts_w[5];
  float* pts_b[5];
  float* fcc_w[5];
  float* fcc_b[5];
  float* out_w;
  float* out_b;
} XrdNiceDecoderGrads;

typedef struct {
  const float* data; /* DEVICE [Z][Y][X][32] */
  int nx, ny, nz;
} XrdNiceGrid;

typedef enum { XRD_NICE_MIDDLE = 0, XRD_NICE_FINE = 1, XRD_NICE_COLOR = 2 } XrdNiceStage;

typedef struct {
  int stage;              /* XrdNiceStage                                          */
  int is_mapping;         /* loss form (conv_onet.py:160-185)                      */
  int n_samples;          /* 32 uniform                                            */
  int n_surface;          /* 16 near the surface                                   */
  double bound_min[3];    /* scene bound AFTER load_bound (float64)                */
  double bound_max[3];
  float w_color;          /* tracking 0.5 / mapping 0.2                            */
  int handle_dynamic;     /* tracking: 10 x median mask                            */
  int use_color_in_tracking;
  const float* t_uniform; /* DEVICE [n_samples] torch.linspace(0,1,n_samples)       */
  const float* t_surface; /* DEVICE [n_surface] torch.linspace(0,1,n_surface)       */
  const float* max_depth_global; /* DEVICE scalar: max(target_d) over the all-rank batch
                           * under data-parallel mapping (far clamp and zero-depth
                           * sampling are batch-global, SURVEY Q9); NULL -> computed
                           * from this call's rays                                  */
} XrdNiceCfg;

typedef struct {
  float* rgb;         /* [R,3]                                                     */
  double* depth;      /* [R]   float64 like the reference                          */
  double* uncertainty;/* [R]                                                       */
  double* z_vals;     /* [R,S] optional                                            */
  float* raw;         /* [R,S,4] optional (rgb, occupancy logit)                   */
  float* losses;      /* [2] depth_loss, rgb_loss (rgb 0 when the stage has none)  */
} XrdNiceOut;

typedef struct {
  float* d_grid[3];            /* middle, fine, color: [Z][Y][X][32], ACCUMULATED;
                                * NULL entries are skipped                         */
  XrdNiceDecoderGrads* d_color;/* colour-decoder gradients or NULL (frozen)         */
  float* d_rays_o;             /* [R,3] or NULL                                     */
  float* d_rays_d;             /* [R,3] or NULL                                     */
} XrdNiceGrads;

size_t xrd_nice_workspace_bytes(int n_rays, int n_samples_total, int with_grads);

/* decoders[3] = middle, fine, color; grids[3] = middle, fine, color. */
int xrd_nice_step(const XrdRays* rays, const XrdNiceGrid grids[3],
                  const XrdNiceDecoder decoders[3], const XrdNiceCfg* cfg,
                  XrdNiceOut* out, XrdNiceGrads* grads, void* workspace,
                  size_t workspace_bytes, void* stream);

/* Mesher queries (slam/models/conv_onet.py:213-240 query_fn = NICE.forward(stage 'fine'),
 * color_func = stage 'color'; slam/common/mesher.py:138-167): raw [P,4] = (rgb or 0, occupancy
 * logit middle [+ fine]) at free points DEVICE [P,3] fp32; no out-of-bound masking (the mesher
 * applies its own). */
size_t xrd_nice_query_workspace_bytes(int n_points);
int xrd_nice_query(const float* points, int n_points, const XrdNiceGrid grids[3],
                   const XrdNiceDecoder decoders[3], const double bound_min[3],
                   const double bound_max[3], int stage, float* raw, void* workspace,
                   size_t workspace_bytes, void* stream);

/* Stage 'coarse' (slam/models/conv_onet.py:137-138 target_d = None, :397-402 near = 0.01 /
 * far = bound exit, 32 uniform samples; slam/model_components/decoder_nice.py:237-320
 * MLP_no_xyz, :389-393): its own decoder and grid; the grid is sampled with the scene bound
 * multiplied by model_coarse_bound_enlarge (conv_onet.py:335-337) while the out-of-bound mask
 * and the far plane use the scene bound.  Mapping depth loss only (conv_onet.py:176-181);
 * the decoder is frozen, gradients go to the grid (ACCUMULATED into d_grid) and the rays. */
typedef struct {
  const float* pts_w[5]; /* DEVICE [32,32] x3, [32,64] (input = [feature, hidden]), [32,32] */
  const float* pts_b[5]; /* DEVICE [32]                                                    */
  const float* out_w;    /* DEVICE [1,32]                                                  */
  const float* out_b;    /* DEVICE [1]                                                     */
} XrdNiceCoarseDecoder;

typedef struct {
  int n_samples;               /* 32                                                      */
  double bound_min[3];         /* scene bound after load_bound                            */
  double bound_max[3];
  double coarse_bound_min[3];  /* scene bound * model_coarse_bound_enlarge                */
  double coarse_bound_max[3];
  const float* t_uniform;      /* DEVICE [n_samples] torch.linspace(0,1,n_samples)        */
} XrdNiceCoarseCfg;

size_t xrd_nice_coarse_workspace_bytes(int n_rays, int n_samples, int with_grads);
/* out->losses[0] = depth loss (losses[1] = 0).  with_grads = 0: forward only. */
int xrd_nice_coarse_step(const XrdRays* rays, const XrdNiceGrid* grid,
                         const XrdNiceCoarseDecoder* dec, const XrdNiceCoarseCfg* cfg,
                         XrdNiceOut* out, float* d_grid, float* d_rays_o, float* d_rays_d,
                         int with_grads, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Vox-Fusion -------------------------------------------------------------
 *
 * Map structure (host side, once per mapping call -- SURVEY row f2):
 *   xrd_octree_*   third_party/sparse_octree: Octree::init/insert
 *                  (src/octree.cpp:35-115), get_centres_and_children (:297-346); node ids
 *                  (= embedding rows, SURVEY Q4) follow the reference's creation order.
 * The octree handle is a host object that owns its memory (like svo.Octree). */
typedef struct XrdOctree XrdOctree;
XrdOctree* xrd_octree_create(int grid_dim); /* 256; NULL on failure                 */
void xrd_octree_destroy(XrdOctree* t);
int xrd_octree_num_nodes(const XrdOctree* t);
/* voxels: HOST int32 [n][3] voxel coordinates (floor(p / voxel_size)); returns the node
 * count after the insertion (negative XrdStatus on error). */
int xrd_octree_insert(XrdOctree* t, const int32_t* voxels, int n);
/* HOST outputs sized by xrd_octree_num_nodes: voxels f32 [N][4], children f32 [N][8],
 * features i32 [N][8].  Returns N. */
int xrd_octree_export(const XrdOctree* t, float* voxels, float* children, int32_t* features);

/* Per-iteration path:
 *   xrd_voxfusion_march   slam/model_components/voxel_helpers_voxfusion.py:647-687 ray_intersect
 *                         (third_party/sparse_voxels/src/intersect_gpu.cu:191-270
 *                         svo_intersect_point_kernel + the host-side fill/sort/trim) and
 *                         :690-714 ray_sample (src/sample_gpu.cu:133-239
 *                         inverse_cdf_sampling_kernel incl. its batching quirks).
 *   xrd_voxfusion_render  slam/models/sparse_voxel.py:152-274 render_rays after sampling:
 *                         get_features (voxel_helpers_voxfusion.py:106-123,147-153), Decoder
 *                         (slam/model_components/decoder_voxfusion.py:122-149), sdf2weights
 *                         (:276-304), get_loss_dict (:103-143, utils.py:154-186) + backward.
 * The two calls are separated by ONE host read of `XrdVoxMarch.stats` (the reference syncs at
 * the same place: `hits.sum() == 0` -> None, sparse_voxel.py:179-181): the render workspace is
 * sized by the number of valid sample points. */
typedef struct {
  int n_nodes;
  const float* centres;      /* DEVICE [N][3]  (xyz + side/2) * voxel_size               */
  const int32_t* children;   /* DEVICE [N][9]  8 child ids (-1: none) ++ side            */
  const int32_t* vertex_idx; /* DEVICE [N][8]  corner-leaf ids = embedding rows          */
  const float* embeddings;   /* DEVICE [n_embeddings][16]                                */
  int n_embeddings;
} XrdVoxMap;

typedef struct {
  float voxel_size;   /* 0.2                                                              */
  float step_size;    /* voxel_size * 0.05 = 0.01 m                                       */
  int max_hits;       /* 50 (ray_intersect's max_hits_temp)                               */
  float max_distance; /* 10                                                               */
  int max_samples;    /* capacity per ray of the sample arrays (>= batch max + hits)      */
  int rays_per_block; /* inverse_cdf batching: K = ceil(R' / 200) of the reference
                         wrapper (voxel_helpers_voxfusion.py:411-424); 0 = derive       */
  uint64_t seed;      /* Philox when noise == NULL                                        */
} XrdVoxMarchCfg;

typedef struct {
  /* sorted, trimmed intersections (DEVICE) */
  int32_t* hit_idx;   /* [R][max_hits]                                                    */
  float* hit_tmin;    /* [R][max_hits]                                                    */
  float* hit_tmax;    /* [R][max_hits]                                                    */
  /* samples (DEVICE) */
  int32_t* smp_idx;   /* [R][max_samples]  voxel id or -1                                 */
  float* smp_depth;   /* [R][max_samples]                                                 */
  float* smp_dist;    /* [R][max_samples]                                                 */
  int32_t* smp_count; /* [R]  valid samples of the ray                                    */
  int32_t* smp_base;  /* [R]  first slot of the ray in the compact point list            */
  uint8_t* ray_mask;  /* [R]  ray hit at least one voxel                                  */
  int32_t* stats;     /* DEVICE [8 + 2R]: 0 n_hit_rays, 1 n_points, 2 S_max (batch max
                         samples), 3 P_max (batch max hits), 4 overflow (samples dropped by
                         the cap); [8, 8+R) rank of each ray among the hit rays, [8+R, 8+2R)
                         rank -> ray                                                       */
} XrdVoxMarch;

/* noise: DEVICE [R][max_samples] uniform(0,1) (clamped to [0.001,0.999] inside) or NULL. */
int xrd_voxfusion_march(const XrdRays* rays, const XrdVoxMap* map, const XrdVoxMarchCfg* cfg,
                        const float* noise, XrdVoxMarch* out, void* stream);

/* Parity hooks: the raw kernels with the reference kernels' exact signatures of data.
 * intersect: unsorted DFS-order hits (idx -1 padded), as svo_intersect returns them.
 * sample: explicit probs / steps / noise, compact layout [R][H] -> [R][max_steps]. */
int xrd_voxfusion_intersect_raw(const XrdRays* rays, const XrdVoxMap* map, float voxel_size,
                                int n_max, int32_t* idx, float* tmin, float* tmax, void* stream);
int xrd_voxfusion_sample_raw(int n_rays, int max_hits, int max_steps, int rays_per_block,
                             const int32_t* pts_idx, const float* min_depth,
                             const float* max_depth, const float* noise, const float* probs,
                             const float* steps, int32_t* smp_idx, float* smp_depth,
                             float* smp_dist, void* stream);

typedef struct {            /* torch nn.Linear layouts [out][in] + bias, DEVICE            */
  const float *w0, *b0;     /* pts_linears.0   [128][16]                                   */
  const float *w1, *b1;     /* pts_linears.1   [128][128]                                  */
  const float *ws, *bs;     /* sdf_out         [129][128]  (sdf, feat128)                  */
  const float *wc0, *bc0;   /* color_out.0     [128][144]  in = feat128 ++ emb16           */
  const float *wc1, *bc1;   /* color_out.2     [3][128]                                    */
} XrdVoxDecoder;

typedef struct {            /* same shapes, ACCUMULATED into                               */
  float *w0, *b0, *w1, *b1, *ws, *bs, *wc0, *bc0, *wc1, *bc1;
} XrdVoxDecoderGrads;

typedef struct {
  float voxel_size;
  float trunc;        /* training_trunc * sc_factor (0.05)                                */
  float max_depth;    /* loss: valid depth in (0.01, max_dpeth)                           */
  float pad_depth;    /* MAX_DEPTH = 10 that pads z_vals (voxel_helpers_voxfusion.py:11)   */
  float w_rgb, w_depth, w_sdf, w_fs; /* .5, 1, 5000, 10                                   */
  int n_points;       /* host copy of stats[1]                                            */
  int s_max;          /* host copy of stats[2]                                            */
  int n_hit_rays;     /* host copy of stats[0]                                            */
} XrdVoxRenderCfg;

typedef struct {
  float* rgb;     /* [R,3]  0 for rays without a hit                                      */
  float* depth;   /* [R]                                                                   */
  float* losses;  /* [4] rgb, depth, sdf, fs (weighted)                                    */
} XrdVoxOut;

typedef struct {
  float* d_embeddings;          /* [n_embeddings][16], ACCUMULATED                        */
  XrdVoxDecoderGrads* d_decoder;/* or NULL                                                */
  float* d_rays_o;              /* [R,3] or NULL                                          */
  float* d_rays_d;              /* [R,3] or NULL                                          */
} XrdVoxGrads;

size_t xrd_voxfusion_render_workspace_bytes(int n_rays, int n_points, int with_grads);

int xrd_voxfusion_render(const XrdRays* rays, const XrdVoxMap* map, const XrdVoxMarch* march,
                         const XrdVoxMarchCfg* mcfg, const XrdVoxDecoder* dec,
                         const XrdVoxRenderCfg* cfg, XrdVoxOut* out, XrdVoxGrads* grads,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Forward-only Decoder.get_values at points that carry a voxel (octree node) id, for mesh
 * extraction.  Replaces slam/model_components/voxel_helpers_voxfusion.py:15-94 (get_scores,
 * eval_points) and their get_features / trilinear_interp (:97-166); same arithmetic as the
 * render path (one shared corner / weight routine, the same decoder GEMM chain).
 *   res > 0, LATTICE mode (get_scores): n = number of voxels, vox DEVICE [n] node ids,
 *       lin DEVICE [res] = torch.linspace(-0.5, 0.5, res) in fp32; point (b, i, j, k) is
 *       xyz = lin[(i, j, k)] * voxel_size + centre[vox[b]] (fp32, rounded per operation).
 *       Only the sdf head runs; sdf DEVICE [n][res][res][res] (meshgrid 'ij': i slowest) --
 *       the marching-cubes volume layout.  xyz and rgb must be NULL.
 *   res == 0, POINT mode (eval_points): n points, xyz DEVICE [n][3], vox DEVICE [n] node ids;
 *       rgb DEVICE [n][3] (sigmoid colour), sdf DEVICE [n] or NULL.
 * The workspace is sized for n_points = n * res^3 (lattice) or n (points). */
size_t xrd_voxfusion_query_workspace_bytes(int n_points);
int xrd_voxfusion_query(const XrdVoxMap* map, const XrdVoxDecoder* dec, float voxel_size, int n,
                        const int32_t* vox, int res, const float* lin, const float* xyz,
                        float* sdf, float* rgb, void* workspace, size_t workspace_bytes,
                        void* stream);

/* ---- Marching cubes ---------------------------------------------------------
 *
 *   xrd_mesh_mc_*  slam/common/mesher.py:206-238 (skimage.measure.marching_cubes over the
 *                  Mesher's lattice, on the host after a D2H copy of every value) and
 *                  slam/algorithms/voxfusion.py:250-278 (one skimage call per surface voxel in
 *                  a Python loop).  One implementation for a batch of B independent volumes
 *                  values DEVICE fp32 [B][nx][ny][nz] (x slowest), nx, ny, nz >= 2.
 *
 * Semantics:
 *   - a corner is negative iff v < level; a lattice edge is crossed iff its two corners are on
 *     different sides;
 *   - each crossed edge gets exactly one vertex per volume, shared by every cube using it
 *     (vertices are not shared across volumes);
 *   - position along the edge v0 -> v1 (v0 at the lower lattice index): t = (level - v0) /
 *     (v1 - v0); p = lattice index with t added on the edge's axis; world coordinate
 *     ((p * spacing + shift) * scale) + origin[b], every operation fp32 round-to-nearest;
 *   - vertex order (volume, flat lattice index of the edge's lower endpoint, axis x, y, z),
 *     face order (volume, cube = flat index of its lower lattice point, triangle in the case);
 *   - winding: the right-hand normal of every face points toward larger values (outward for
 *     an SDF that is negative inside).  The case table (csrc/mc_table.cuh) is generated by
 *     oracle/mc_table.py; ambiguous faces separate their two negative corners.
 * Differences from skimage's Lewiner method are expected on ambiguous cubes only (asymptotic
 * decider, extra interior vertex); the reference's two callers map to the affine as
 *   Mesher:     spacing (x[2]-x[1], ...), shift (x[0], y[0], z[0]), scale 1, origin NULL;
 *   Vox-Fusion: spacing 1/(res-1), shift -0.5, scale voxel_size, origin = voxel centres.
 *
 * Two phases: xrd_mesh_mc_count classifies the cubes, scans the per-point vertex and triangle
 * counts into the workspace and writes the totals (V, F) to DEVICE counts[2]; the caller reads
 * them, allocates verts f32 [V][3] and faces i32 [F][3], and calls xrd_mesh_mc_emit with the
 * same values, shape, level and workspace.  Nothing is allocated inside. */
typedef struct {
  float spacing[3];
  float shift[3];
  float scale[3];
  const float* origin;  /* DEVICE [B][3] or NULL (zero)                                   */
} XrdMeshAffine;

size_t xrd_mesh_mc_workspace_bytes(int B, int nx, int ny, int nz);
int xrd_mesh_mc_count(const float* values, int B, int nx, int ny, int nz, float level,
                      int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int xrd_mesh_mc_emit(const float* values, int B, int nx, int ny, int nz, float level,
                     const XrdMeshAffine* affine, float* verts, int32_t* faces, void* workspace,
                     size_t workspace_bytes, void* stream);

/* ---- TSDF fusion (Point-SLAM get_mesh) -----------------------------------------
 *
 *   xrd_tsdf_alloc_*, xrd_tsdf_integrate  slam/common/common.py:622-657 (get_mesh_from_RGBD:
 *                  open3d ScalableTSDFVolume(voxel_length 4/512, sdf_trunc 0.04, RGB8) and one
 *                  volume.integrate per keyframe, on the host)
 *   xrd_tsdf_mc_*  slam/common/common.py:658 (volume.extract_triangle_mesh)
 *   xrd_tsdf_components  slam/common/common.py:666-677 (clean_mesh:
 *                  trimesh.graph.connected_components over the mesh edges)
 *
 * open3d and trimesh are not vendored; the semantics below are this library's own.  Where a
 * choice follows open3d it is marked [from memory -- unverified]; parity with open3d is
 * unpinned.  A numpy restatement (oracle/tsdf.py) matches the kernels bit for bit.
 *
 * Volume.  Blocks of 16^3 voxels, voxel edge vl = voxel_length, block edge bl = 16 * vl
 * [open3d's default block resolution, from memory -- unverified].  Block (bx, by, bz) is keyed
 * by ((bx + 2^20) << 42) | ((by + 2^20) << 21) | (bz + 2^20) (21 signed bits per axis, int64,
 * |b| < 2^20).  Voxel (i, j, k) of a block (x slowest, flat index i*256 + j*16 + k) has the
 * centre b*bl + (i + 0.5)*vl per axis; it stores tsdf f32 (0 initially), weight f32 (0) and
 * colour f32 [3] on the 0..255 scale (0).
 *
 * Inputs.  K frames: depth DEVICE f32 [K][H][W] (0 = invalid; d > depth_trunc counts as 0),
 * colour DEVICE u8 [K][H][W][3], c2w DEVICE f32 [K][3][4] (camera to world, open3d axes: x
 * right, y down, z forward) and w2c DEVICE f32 [K][3][4] (its inverse).  Camera coordinates
 * of pixel (u, v) at depth d: x = ((u - cx) * d) / fx, y = ((v - cy) * d) / fy, z = d.  A
 * [3][4] transform T maps p to ((T[r][0]*p0 + T[r][1]*p1) + T[r][2]*p2) + T[r][3].
 *
 * Allocation.  Every pixel with u % stride == 0, v % stride == 0 and a valid depth is
 * back-projected with c2w to p; per axis the blocks floor((p - sdf_trunc) / bl) ..
 * floor((p + sdf_trunc) / bl) are touched by the frame (at most 2 per axis: 2 * sdf_trunc <
 * bl is required).  Points whose blocks leave the key range are skipped.  The allocated set is
 * the sorted unique union of the touched keys; block ids are ranks in it.  Each block carries a
 * touched-frame bitmask u32 [ceil(K/32)] (bit k%32 of word k/32).
 *
 * Integration [ScalableTSDFVolume semantics: a frame updates only the blocks it touched, from
 * memory -- unverified].  For every voxel of every block, for the block's frames in order:
 *   (x, y, z) = w2c * centre; skip if z <= 0;
 *   u = floor(fx * x / z + cx + 0.5), v = floor(fy * y / z + cy + 0.5) (nearest pixel, halves
 *   up); skip unless 0 <= u < W, 0 <= v < H and the depth d there is valid;
 *   sdf = (d - z) * sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1); skip if sdf <= -sdf_trunc;
 *   t = min(1, sdf / sdf_trunc); tsdf = (tsdf * w + t) / (w + 1); colour = (colour * w +
 *   c_k) / (w + 1) per channel; w = w + 1.
 * Every fp32 operation is rounded to nearest in the order written (no contraction).
 *
 * Extraction.  A cube is anchored at every voxel of every block; its corners (i + di, j + dj,
 * k + dk) with an index of 16 lie in the +x / +y / +z neighbour blocks.  A cube is used iff all
 * 8 corners exist (allocated) with weight > 0; its case comes from csrc/mc_table.cuh with a
 * corner negative iff tsdf < 0.  A crossed edge gets one vertex iff a used cube references it;
 * the vertex belongs to the edge's lower voxel (possibly in a neighbour block), so vertices are
 * shared across block seams.  Along the edge v0 -> v1: t = (0 - v0) / (v1 - v0); position
 * ((c * vl + vl * 0.5) * 1) + b * bl per axis with c the lower voxel's local index plus t on the
 * edge's axis (the mesh.cu affine); colour (c0 + t * (c1 - c0)) / 255.  Vertex order (block id,
 * voxel, axis), face order (block id, voxel, triangle), both from exclusive scans; right-hand
 * normals point toward positive tsdf (free space, the camera).  As with xrd_mesh_mc_*, a cube
 * face whose four edges are crossed can carry a triangle of the case table flat in that face,
 * which the cube on the other side emits reversed (rare: < 0.1% of faces on the synthetic room).
 *
 * Components.  labels[v] = the smallest vertex id connected to v through face edges (v itself
 * for a vertex in no face); deterministic.  faces must index [0, n_verts).
 *
 * Two phases per pass as for xrd_mesh_mc_*: xrd_tsdf_alloc_count writes the block count to
 * DEVICE n_blocks[1]; the caller allocates keys i64 [n_blocks] and masks u32 [n_blocks][ceil(K/
 * 32)] and calls xrd_tsdf_alloc_emit with the same inputs' shape, params and workspace.
 * xrd_tsdf_mc_count writes (V, F) to DEVICE counts[2]; xrd_tsdf_mc_emit fills verts f32 [V][3],
 * colors f32 [V][3] and faces i32 [F][3] from the same keys, tsdf and workspace.  integrate
 * updates tsdf / weight / color_acc ([n_blocks * 4096], [.], [. * 3]) of the blocks in keys in
 * place with the masks' frames; n_blocks * 4096 < 2^31.  Nothing is allocated inside. */
typedef struct {
  float voxel_length;
  float sdf_trunc;
  float depth_trunc;
  float fx, fy, cx, cy;
  int stride; /* allocation samples every stride-th pixel in u and v                    */
} XrdTsdfParams;

size_t xrd_tsdf_alloc_workspace_bytes(int K, int H, int W, int stride);
int xrd_tsdf_alloc_count(const float* depth, const float* c2w, int K, int H, int W,
                         const XrdTsdfParams* params, int32_t* n_blocks, void* workspace,
                         size_t workspace_bytes, void* stream);
int xrd_tsdf_alloc_emit(int K, int H, int W, const XrdTsdfParams* params, int n_blocks,
                        int64_t* keys, uint32_t* masks, void* workspace, size_t workspace_bytes,
                        void* stream);
int xrd_tsdf_integrate(const int64_t* keys, const uint32_t* masks, int n_blocks,
                       const float* depth, const uint8_t* color, const float* w2c, int K, int H,
                       int W, const XrdTsdfParams* params, float* tsdf, float* weight,
                       float* color_acc, void* stream);
size_t xrd_tsdf_mc_workspace_bytes(int n_blocks);
int xrd_tsdf_mc_count(const int64_t* keys, int n_blocks, const float* tsdf, const float* weight,
                      int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int xrd_tsdf_mc_emit(const int64_t* keys, int n_blocks, const float* tsdf,
                     const float* color_acc, const XrdTsdfParams* params, float* verts,
                     float* colors, int32_t* faces, void* workspace, size_t workspace_bytes,
                     void* stream);
int xrd_tsdf_components(const int32_t* faces, int n_faces, int n_verts, int32_t* labels,
                        void* stream);

/* ---- Mesh culling (cull_mesh) ---------------------------------------------------
 *
 *   xrd_cull_visible  slam/common/common.py:714-783 (cull_mesh's per-frame loop: every vertex
 *                     projected into every frame, an H2D copy of the vertices and a D2H copy of
 *                     the mask per frame, ANDed on the host)
 *   xrd_cull_count / xrd_cull_emit  common.py:784-787 (whole_mask[faces].all(1),
 *                     mesh.update_faces, mesh.remove_unreferenced_vertices)
 *
 * Visibility.  verts DEVICE f32 [V][3] (the reference's .float() of the vertices); w2c DEVICE
 * f32 [F][3][4], rows 0..2 of torch.inverse(c2w) of each frame (computed by the caller with that
 * call); depth DEVICE f32 [F][H][W].  A [3][4] row applied to (x, y, z, 1) is ((T0*x + T1*y) +
 * T2*z) + T3.  Per frame: cam = w2c (x, y, z, 1); xc = -cam.x, yc = cam.y, zc = cam.z;
 * u' = fx*xc + cx*zc, v' = fy*yc + cy*zc (K's zero products are left out: a +-0 term changes no
 * decision); z = zc + f32(1e-5); u = u' / z, v = v' / z.  The frame sees the vertex iff
 *   0 <= -z, 0 < u < W, 0 < v < H   and, with eval_rec, d + truncation >= -z,
 * where d = grid_sample(depth, 2 * (u / W, v / H) - 1, bilinear, padding 'zeros',
 * align_corners=True): the source coordinate is ((g + 1) / 2) * (size - 1) per axis (so the
 * pixel sampled is u * (W - 1) / W), corners (floor, floor + 1), weights nw = (x1 - ix) * (y1 -
 * iy), ne = (ix - x0) * (y1 - iy), sw = (x1 - ix) * (iy - y0), se = (ix - x0) * (iy - y0), and
 * d = ((nw*D_nw + ne*D_ne) + sw*D_sw) + se*D_se over the corners inside the image (zeros
 * padding; invalid pixels, depth 0, take part).  [torch's scalar unnormalise and blend order,
 * from memory -- unverified; torch's own kernels may contract or reorder, so bit parity with
 * torch is unpinned.]  Every fp32 operation is rounded to nearest in the order written (no
 * contraction).  The frustum tests come first: depth is read only for a vertex inside the image;
 * behind the camera, at z ~ 0 and with a non-finite u or v the tests are false.
 * seen u8 [V] is OR-ed in place (set to 1, never cleared); vertices already seen are skipped,
 * so the result does not depend on how the frames are split over calls.  1 <= F <=
 * XRD_CULL_MAX_FRAMES (the poses are staged in shared memory).
 *
 * Compaction.  A face is kept iff one of its vertices is seen (the reference removes the faces
 * whose three vertices are all unseen); a vertex is kept iff a kept face references it (a seen
 * vertex in no kept face is dropped, an unseen vertex of a kept face stays).  Both keep their
 * order; faces are remapped to the kept vertices; colours (color_bytes bytes per vertex, any
 * element type, or 0 = none) follow their vertices.  trimesh's tolerance merge in
 * mesh.process(validate=False) is not reproduced (culling creates no new duplicates).
 * xrd_cull_count writes (V', F', n_bad) to DEVICE counts[3], n_bad = faces with an index
 * outside [0, V) (neither kept nor read; the caller treats n_bad > 0 as an error); the caller
 * allocates verts f32 [V'][3], faces i32 [F'][3] and colours u8 [V'][color_bytes] and calls
 * xrd_cull_emit with the same sizes and workspace (any output may be NULL).  Nothing is allocated
 * inside. */
#define XRD_CULL_MAX_FRAMES 1024
typedef struct {
  int H, W;
  float fx, fy, cx, cy; /* rounded to f32 like the reference's K.float()                      */
  float truncation;     /* f32, default 0.06                                                  */
  int eval_rec;         /* 0: the depth term is dropped                                       */
} XrdCullParams;

int xrd_cull_visible(const float* verts, int n_verts, const float* w2c, const float* depth,
                     int n_frames, const XrdCullParams* params, uint8_t* seen, void* stream);
size_t xrd_cull_workspace_bytes(int n_verts, int n_faces);
int xrd_cull_count(const uint8_t* seen, int n_verts, const int32_t* faces, int n_faces,
                   int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int xrd_cull_emit(const float* verts, const uint8_t* colors, int color_bytes, int n_verts,
                  const int32_t* faces, int n_faces, float* out_verts, uint8_t* out_colors,
                  int32_t* out_faces, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Reconstruction metrics (ds-eval) -------------------------------------------
 *
 *   xrd_eval_surface_* scripts/utils/eval_recon.py:120-124 (trimesh.sample.sample_surface) and
 *                      evaluate_3d_reconstruction.py:182-201 (open3d sample_points_uniformly)
 *   xrd_nn_*           eval_recon.py:29-47 (scipy cKDTree queries), open3d's
 *                      compute_point_cloud_distance (evaluation.py:78-82) and the KD-tree
 *                      correspondences of open3d's point-to-point registration_icp
 *   xrd_eval_*_stats   the means / counts of those distances and ICP's correspondence sums
 *   xrd_eval_transform trimesh's apply_transform of the mesh vertices
 *
 * Surface sampling.  xrd_eval_surface_prepare: verts DEVICE f32 [V][3], faces DEVICE i32 [F][3]
 * (F >= 1, V >= 1, else XRD_E_SHAPE at once).  Face areas are float64: with a = v0 and the fp32
 * coordinates widened exactly, e1 = v1 - a, e2 = v2 - a, c = e1 x e2 (each component
 * e1y*e2z - e1z*e2y etc.), area = 0.5 * sqrt((cx*cx + cy*cy) + cz*cz).  cum DEVICE f64 [F] is
 * their inclusive prefix in chunks of XRD_EVAL_AREA_CHUNK faces: sequential inside a chunk,
 * plus the chunk's offset (the sequential sum of the earlier chunks' totals) in one final add
 * (off + local); total DEVICE f64 [1] = the sum of the chunk totals.  status DEVICE i32 [1]
 * becomes XRD_E_SHAPE when a vertex coordinate is not finite, a face index lies outside
 * [0, V) (its area is not read) or the total is not finite and > 0; 0 otherwise.  The caller
 * reads status and treats a non-zero value as the call's error; xrd_eval_sample_surface writes
 * nothing while status is non-zero, so it never reads a bad face.
 * xrd_eval_sample_surface writes out f32 [n][3] (and face_ids i32 [n], optional):
 *   XRD_EVAL_TRIMESH (trimesh sample_surface; from memory, unverified): uniforms [n][3] =
 *     (u0, u1, u2); face = first t with cum[t] >= u0 * total (f64; searchsorted 'left',
 *     clamped to F - 1); if u1 + u2 > 1 (fp32) both become |u - 1|;
 *     p = v0 + (u1 * (v1 - v0) + u2 * (v2 - v0)) per axis in fp32.
 *   XRD_EVAL_OPEN3D (open3d sample_points_uniformly; from memory, unverified): sample k belongs
 *     to the first face t with round((cum[t] / total) * n) > k (f64, round half away from
 *     zero), so face t receives [round(C_{t-1} n), round(C_t n)) deterministically;
 *     uniforms [n][2] = (r1, r2); s = sqrt(r1), a = 1 - s, b = s * (1 - r2), c = s * r2;
 *     p = (a * v0 + b * v1) + c * v2 per axis in fp32.
 * uniforms DEVICE f32 (parity mode) or NULL: then sample k draws philox4(seed, k) (common.cuh)
 * and uses its first three (two) values.  The reference's draws are unseeded and its prefix
 * sums are sequential, so the metrics are statistically equivalent to the reference's, not
 * equal.  All fp32 / fp64 operations round to nearest in the order written.
 *
 * Exact nearest neighbour.  An index over target points P [N][3] is a dense grid over their
 * bounding box: xrd_nn_layout (host, deterministic in N and the f64 box) picks the smallest cell
 * h (64-step bisection) with prod_a (floor(ext_a / h) + 1) <= 2N cells and at most
 * XRD_NN_MAX_DIM per axis, so the index is O(N); a box of zero extent gets h = 1 and one cell.
 * Above the cells sit n_levels occupancy levels of an implicit octree (level l has
 * ceil(dims / 2^l) nodes per axis, up to one root node).  xrd_nn_build bins every point by
 * floor((x - origin) * inv_h) (fp32, clamped to the grid), radix-sorts (cell, id) so ids
 * ascend inside a cell, and writes cell_ptr [n_cells + 1] (exclusive prefix of the counts),
 * sorted f32 [N][4] = (x, y, z, id as int bits) and occ u8 [occ_bytes].  The caller allocates
 * those three after xrd_nn_layout and reads the box once on the host.
 * xrd_nn_query: for each query q the nearest target by
 *   dx = q - p (fp32), d2 = (dx*dx + dy*dy) + dz*dz (fp32, round to nearest, no FMA),
 *   ties on d2 to the smallest target id; dist = sqrt_rn(d2), ids = the target id.
 * radius <= 0 or infinite: unbounded.  radius > 0: only targets with d2 <= fl(radius * radius)
 * qualify; with none, ids = -1 and dist = +inf.  The search descends the octree near-first and
 * skips a node whose box (padded by `pad`, larger than any rounding of the binning) lies
 * further than the best d2 with a relative margin of 2e-5, so the result is the minimum of
 * (d2, id) over all targets whatever the order and however the queries are split over calls.
 * Queries outside the box start at the root like any other; work is bounded by the occupied
 * nodes near the answer, not by the empty space in between.
 *
 * Reductions.  Element i of n goes to partial i / XRD_EVAL_RED_CHUNK; inside a partial thread
 * t (of 256) sums its elements in index order, then a fixed shared-memory tree; the partials
 * are summed in index order.  All sums are f64 (round to nearest), so a result is
 * bit-identical run to run and depends only on the element values.
 * xrd_eval_dist_stats: out DEVICE f64 [3] = (sum d, sum d*d, count of d < tau in fp32).
 * xrd_eval_icp_stats: for each i with ids[i] >= 0 (s = src[i], t = tgt[ids[i]], both widened
 * exactly to f64): out DEVICE f64 [17] = (count, sum s [3], sum t [3], sum s_a t_b [3][3]
 * row-major, sum d*d).  Both take workspace >= xrd_eval_reduce_workspace_bytes(n).
 * xrd_eval_transform: out = fp32(((T0 x + T1 y) + T2 z) + T3) per row, computed in f64 with
 * the fp32 input widened exactly; T HOST f64 [3][4] (rows 0..2 of the 4x4, row-major), read
 * before the call returns.  out may alias points.
 * xrd_debug_nn_counters: DEVICE u64 [2] or NULL; when set, every later xrd_nn_query on this
 * thread adds (octree nodes entered, target points tested) into it (thread-local, like the
 * error state).  Nothing is allocated inside. */
#define XRD_EVAL_AREA_CHUNK 256
#define XRD_EVAL_RED_CHUNK 4096
#define XRD_EVAL_TRIMESH 0
#define XRD_EVAL_OPEN3D 1
#define XRD_NN_MAX_DIM 32768
#define XRD_NN_MAX_LEVELS 16
typedef struct {
  float origin[3];             /* f32(bbox_min)                                             */
  float h, inv_h;              /* cell edge, f32(1 / h)                                     */
  float pad;                   /* node boxes are widened by this much on every side         */
  int dims[3];                 /* cells per axis                                            */
  int n_cells, n_levels;       /* n_levels: octree levels above the cells (0 = one cell)    */
  int level_off[XRD_NN_MAX_LEVELS]; /* offset of level l (1..n_levels) in occ             */
  int occ_bytes;
  int n_points;
  const int32_t* cell_ptr;     /* DEVICE [n_cells + 1]                                      */
  const uint8_t* occ;          /* DEVICE [occ_bytes] (may be NULL when n_levels == 0)       */
  const float* sorted;         /* DEVICE [n_points][4], 16-byte aligned                     */
} XrdNnIndex;

size_t xrd_eval_surface_workspace_bytes(int n_faces);
int xrd_eval_surface_prepare(const float* verts, int n_verts, const int32_t* faces, int n_faces,
                             double* cum, double* total, int32_t* status, void* workspace,
                             size_t workspace_bytes, void* stream);
int xrd_eval_sample_surface(const float* verts, const int32_t* faces, int n_faces,
                            const double* cum, const double* total, const int32_t* status,
                            int mode, int n_samples, const float* uniforms, uint64_t seed,
                            float* out, int32_t* face_ids, void* stream);
int xrd_nn_layout(int n_points, const double* bbox_min, const double* bbox_max,
                  XrdNnIndex* index);
size_t xrd_nn_build_workspace_bytes(const XrdNnIndex* index);
int xrd_nn_build(const float* points, const XrdNnIndex* index, void* workspace,
                 size_t workspace_bytes, void* stream);
int xrd_nn_query(const XrdNnIndex* index, const float* queries, int n_queries, float radius,
                 float* dist, int32_t* ids, void* stream);
int xrd_debug_nn_counters(unsigned long long* counters);
size_t xrd_eval_reduce_workspace_bytes(int n);
int xrd_eval_dist_stats(const float* dist, int n, float tau, double* out, void* workspace,
                        size_t workspace_bytes, void* stream);
int xrd_eval_icp_stats(const float* src, const float* tgt, const int32_t* ids, const float* dist,
                       int n, double* out, void* workspace, size_t workspace_bytes, void* stream);
int xrd_eval_transform(const float* points, int n, const double* T, float* out, void* stream);

/* ---- Depth L1 (ds-eval calc_2d_metric) -----------------------------------------
 *
 *   xrd_eval_render_depth  eval_recon.py:234-265: open3d Visualizer depth captures of a mesh
 *                          (mesh_show_back_face, constant z_far 20, capture_depth_float_buffer)
 *   xrd_eval_points_seen   eval_recon.py:66-90 check_proj, for many candidate views at once
 *   xrd_eval_depth_l1      eval_recon.py:267-274: per view |gt - rec| over rec > 0
 *
 * Depth rasteriser.  verts DEVICE f32 [V][3], faces DEVICE i32 [F][3], w2c DEVICE f64
 * [n_views][3][4] (rows 0..2 of world-to-camera, OpenCV: +z forward, +y down),
 * 1 <= n_views <= XRD_EVAL_RENDER_MAX_VIEWS, F * n_views < 2^31.  depth DEVICE f32
 * [n_views][H][W] is written whole: the nearest fragment's z, 0 where nothing is drawn.
 * Per view and face (no culling; open3d's behaviour restated from memory, unverified):
 *   1. camera space in f64: p = ((r0 x + r1 y) + r2 z) + t per row, x y z the fp32 vertex.
 *   2. a face whose three z are all < z_near draws nothing.  Otherwise the triangle is clipped
 *      (Sutherland-Hodgman, vertex order kept) against z >= z_near, then against the guard band
 *      |fx x| <= G z and |fy y| <= G z, G = XRD_EVAL_RENDER_GUARD pixels, in that order.  A
 *      crossing on segment (a, b) is computed from its lexicographically (x, y, z) smaller end:
 *      t = d_a / (d_a - d_b), p = a + t (b - a), so faces sharing an edge share the point even
 *      when their vertices are duplicates.  The polygon is fanned as (0, k, k + 1).
 *   3. each vertex projects to u = (fx x) / z + cx, v = (fy y) / z + cy (f64) and snaps to
 *      X = rint(256 u), Y = rint(256 v) (int64, 1/XRD_EVAL_RENDER_SUBPIXEL pixel).  Pixel (i, j)
 *      samples (256 i, 256 j), i.e. u = i, v = j (GL's pixel centre when cx = W / 2 - 0.5).
 *      A triangle with zero snapped area draws nothing; otherwise pixel (i, j) is covered when
 *      its three int64 edge functions are all >= 0 (area > 0) or all <= 0 (area < 0), so a
 *      pixel on a shared edge is drawn by both faces and a closed surface has no cracks.
 *   4. depth is perspective-correct from the unclipped face's plane: n = (p1 - p0) x (p2 - p0),
 *      k = (n_x p0_x + n_y p0_y) + n_z p0_z (f64), ax = n_x / fx, ay = n_y / fy,
 *      c0 = n_z - (ax cx + ay cy), z = fp32(k / ((ax i + ay j) + c0)).  k = 0 draws nothing; a
 *      fragment is kept when 0 < z <= fp32(z_far) and z is finite.  The image keeps the
 *      smallest z (an integer max on the complemented bits), so it does not depend on the order
 *      of faces or on the launch split.
 * Faces whose pixel box has more than XRD_EVAL_RENDER_INLINE_PX pixels, or that need clipping,
 * are queued in the workspace and drawn by one warp each; the result is the same either way.
 * status DEVICE i32 [1] becomes XRD_E_SHAPE when a face index lies outside [0, V) (depth is
 * then undefined), 0 otherwise.  H, W <= XRD_EVAL_RENDER_MAX_SIDE, fx, fy > 0,
 * 0 < z_near < z_far, |cx|, |cy| <= 2 XRD_EVAL_RENDER_MAX_SIDE, else XRD_E_SHAPE at once.
 * Workspace >= xrd_eval_render_workspace_bytes(F, n_views) (4 bytes per (face, view) + 256).
 * xrd_debug_eval_render_queued: *count (DEVICE u32) = the faces the last render with this
 * workspace queued, summed over its views.
 *
 * Unseen check.  xrd_eval_points_seen: points DEVICE f32 [N][3], w2c DEVICE f32 [K][3][4] =
 * fp32(inv(c2w with columns 1 and 2 negated)) as check_proj builds it; seen DEVICE u8 [K].
 * In fp32, per point and view: c = ((w0 x + w1 y) + w2 z) + w3 per row; x' = -c_x;
 * u' = fx x' + cx c_z, v' = fy c_y + cy c_z; z' = c_z + fp32(1e-5); u = u' / z', v = v' / z';
 * seen[k] = 1 when some point has 0 <= -z', 0 < u < W and 0 < v < H (fx..cy, W, H as fp32).
 * The reference multiplies with torch matmuls whose summation order is unspecified.
 *
 * Per-view sums.  xrd_eval_depth_l1: gt, rec DEVICE f32 [n_views][n_pixels]; out DEVICE f64
 * [n_views][2] = (sum |gt - rec|, count) over the pixels with rec > 0.  The fp32 difference is
 * widened exactly; thread t of 256 sums pixels t, t + 256, ... in order, then a fixed tree, so
 * the sums are bit-identical run to run.  The reference takes the mean in fp32 numpy. */
#define XRD_EVAL_RENDER_MAX_VIEWS 32
#define XRD_EVAL_RENDER_SUBPIXEL 256
#define XRD_EVAL_RENDER_INLINE_PX 64
#define XRD_EVAL_RENDER_GUARD 2097152.0
#define XRD_EVAL_RENDER_MAX_SIDE 16384
typedef struct {
  int H, W;
  double fx, fy, cx, cy;
  double z_near, z_far;
} XrdEvalCamera;

size_t xrd_eval_render_workspace_bytes(int n_faces, int n_views);
int xrd_eval_render_depth(const float* verts, int n_verts, const int32_t* faces, int n_faces,
                          const double* w2c, int n_views, const XrdEvalCamera* camera,
                          float* depth, int32_t* status, void* workspace, size_t workspace_bytes,
                          void* stream);
int xrd_debug_eval_render_queued(const void* workspace, unsigned* count, void* stream);
int xrd_eval_points_seen(const float* points, int n_points, const float* w2c, int n_views,
                         const XrdEvalCamera* camera, uint8_t* seen, void* stream);
int xrd_eval_depth_l1(const float* gt, const float* rec, int n_views, int n_pixels, double* out,
                      void* stream);

/* ---- Render-quality metrics of re-rendered frames ------------------------------
 *
 *   xrd_eval_image_metrics  slam/common/common.py:429-479 save_render_imgs: clip, the colour
 *                           mask when no depth is rendered, F.mse_loss / PSNR, the masked
 *                           rendered-depth L1 and pytorch_msssim.ms_ssim(data_range=1,
 *                           size_average=True), for B frames per call; called once per
 *                           re-rendered frame by slam/pipeline/tracker.py:343-409
 *                           save_re_render_frames.  LPIPS is not computed here.
 *
 * gt_color, color DEVICE f32 [B][H][W][3]; gt_depth DEVICE f32 [B][H][W]; depth DEVICE f64
 * [B][H][W] (render_img's depth is float64).  flags: XRD_EVAL_IMAGE_NO_DEPTH = no rendered
 * depth (depth is ignored and may be NULL).  out DEVICE f64 [B][XRD_EVAL_IMAGE_OUT] = (psnr,
 * ms_ssim, depth_l1, mse); levels DEVICE f64 [B][5][3][2] = (mean ssim, mean cs) per level and
 * channel, or NULL.  Per frame, in this order:
 *   1. colour: both images are clipped to [0, 1] (fminf(fmaxf(v, 0), 1)).  With NO_DEPTH both
 *      are then multiplied by (gt_depth > 0) (common.py:447-450); otherwise they are not masked.
 *   2. mse: the fp32 squared difference (a - r)^2 of every element, widened to f64 and summed;
 *      mse = sum / (3 H W); psnr = -10 log10(mse) (+inf when mse = 0).
 *   3. depth_l1 = 100 (sum |(f64) gt - r| / count) over the pixels with gt > 0, all f64; NaN
 *      when there is none.  0 with NO_DEPTH (common.py:460).
 *   4. ms_ssim, five levels l = 0..4 of an image pyramid, per channel, all in fp32 with every
 *      operation rounded in the order written (no contraction):
 *      - window w[11]: d = k - 5, g_k = fp32(exp(fp32(-(d d) / 4.5))), s = g_0 + ... + g_10 summed
 *        in order, w_k = g_k / s.
 *      - filter: valid (unpadded) 11-tap correlation along x (columns) first, then along y (rows),
 *        each as ((w_0 v_0 + w_1 v_1) + ...) + w_10 v_10, of the five maps x, y, x x, y y, x y
 *        (x = gt, y = render; the products are formed before filtering).  A level of H_l x W_l
 *        gives (H_l - 10) x (W_l - 10) outputs.
 *      - from mu1, mu2 and the filtered squares: s1 = E[x x] - mu1 mu1, s2 = E[y y] - mu2 mu2,
 *        s12 = E[x y] - mu1 mu2, cs = (2 s12 + C2) / ((s1 + s2) + C2),
 *        ssim = ((2 mu1 mu2 + C1) / ((mu1 mu1 + mu2 mu2) + C1)) cs, C1 = fp32(0.01^2),
 *        C2 = fp32(0.03^2).  Their means over the valid outputs are f64: each 32 x 16 output
 *        tile is summed by 256 threads (thread t = 32 r + q takes rows r and r + 8 of column q,
 *        in that order), then a fixed tree over the threads; the tile sums of a level are summed
 *        thread t taking tiles t, t + 256, ... in order, then the same tree; mean = sum / count.
 *      - pooling to the next level: avg_pool2d(kernel 2, stride 2, padding s % 2 per axis,
 *        count_include_pad): H_{l+1} = (H_l + 1) / 2, output (i, j) = (((v00 + v01) + v10) + v11)
 *        * 0.25 over input rows 2i - H_l % 2 + {0, 1} and columns 2j - W_l % 2 + {0, 1}, zeros
 *        outside.
 *      - ms_ssim = mean over the 3 channels of prod_l p_l (left to right), p_l = pow(relu(cs_l),
 *        w_l) for l < 4 and pow(relu(ssim_4), w_4), weights fp32(0.0448, 0.2856, 0.3001,
 *        0.2363, 0.1333) widened to f64; the channel mean is ((c0 + c1) + c2) / 3, all f64.
 *      The reference passes the image transposed, [1, 3, W, H]; its filter runs along W first
 *      too, and the window and pooling are symmetric in the axes, so the transposition only
 *      changes the order in which the 2x2 pooling windows and the means are summed.
 * The frame sums of steps 2 and 3 are fixed-order: 256 threads per chunk of 4096 pixels, thread
 * t summing pixels t, t + 256, ... (channels 0, 1, 2 of each) in order, a fixed tree, then the
 * chunk sums as the tile sums above.  Everything is bit-identical run to run.
 * min(H, W) >= XRD_EVAL_IMAGE_MIN_SIDE (pytorch_msssim asserts min(H, W) > (11 - 1) 2^4),
 * max(H, W) <= XRD_EVAL_IMAGE_MAX_SIDE, 1 <= B <= 65535 and no unknown flag, else XRD_E_SHAPE;
 * a required pointer NULL: XRD_E_NULL; workspace < xrd_eval_image_workspace_bytes(B, H, W):
 * XRD_E_WORKSPACE. */
#define XRD_EVAL_IMAGE_LEVELS 5
#define XRD_EVAL_IMAGE_MIN_SIDE 161
#define XRD_EVAL_IMAGE_MAX_SIDE 16384
#define XRD_EVAL_IMAGE_NO_DEPTH 1
#define XRD_EVAL_IMAGE_OUT 4
size_t xrd_eval_image_workspace_bytes(int B, int H, int W);
int xrd_eval_image_metrics(const float* gt_color, const float* color, const float* gt_depth,
                           const double* depth, int B, int H, int W, int flags, double* out,
                           double* levels, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Point-SLAM -------------------------------------------------------------
 *
 *   xrd_pointslam_knn_query  slam/model_components/neural_point_cloud.py:223-282
 *                            find_neighbors_faiss.  The reference's index is faiss-gpu
 *                            IndexIVFFlat(nlist 400, nprobe 4) -- approximate, un-vendored;
 *                            this is an EXACT radius-limited 8-NN (ties by lower id) over a
 *                            uniform hash grid, with faiss's sentinels (id -1, D = FLT_MAX).
 *   xrd_pointslam_step       slam/models/conv_onet_pointslam.py:311-461 render_batch_ray
 *                            (5 surface samples), :248-309 eval_points, POINT.forward
 *                            slam/model_components/decoder_pointslam.py:595-655 stage
 *                            'geometry' (MLP_geometry :162-273: inverse-distance kNN feature
 *                            interpolation + 5x32 Fourier MLP) and stage 'color' (adds
 *                            MLP_color :408-542 with the per-neighbour MLP_col_neighbor
 *                            :276-292), raw2outputs_nerf_color2
 *                            slam/model_components/utils.py:247-295, get_loss_dict
 *                            conv_onet_pointslam.py:144-195 and autograd's backward.
 */
typedef struct {
  const float* pos;           /* DEVICE [N][3] neural point positions                      */
  int n_points;
  float cell;                 /* grid cell edge (>= the largest query radius / 2)          */
  int table_size;             /* power of two                                              */
  const int32_t* cell_start;  /* DEVICE [table_size] first slot of the bucket              */
  const int32_t* cell_end;    /* DEVICE [table_size] one past the last slot                */
  const int32_t* sorted_ids;  /* DEVICE [N] point ids ordered by bucket                    */
} XrdPointIndex;

/* bucket of cell (ix,iy,iz): ((ix*73856093) ^ (iy*19349663) ^ (iz*83492791)) & (table-1),
 * uint32 arithmetic, ix = floor(x * (1/cell)).
 * xrd_pointslam_knn_build fills cell_start / cell_end [table_size] and sorted_ids [n_points]
 * (ids ascending inside a bucket) for DEVICE positions [n_points,3] -- what faiss's
 * index.add() does in the reference (slam/model_components/neural_point_cloud.py:48-52,
 * 173-176), on the device with no host round trip. */
size_t xrd_pointslam_knn_build_workspace_bytes(int table_size);
int xrd_pointslam_knn_build(const float* pos, int n_points, float cell, int table_size,
                            int32_t* cell_start, int32_t* cell_end, int32_t* sorted_ids,
                            void* workspace, size_t workspace_bytes, void* stream);
int xrd_pointslam_knn_query(const XrdPointIndex* index, const float* queries, const float* radius,
                            int radius_stride, int n_queries, float* D, int32_t* I,
                            int32_t* neighbor_num, void* stream);

typedef struct {
  int stage;               /* 0 = 'geometry', 1 = 'color'                                   */
  int is_mapping;
  int n_surface;           /* 5                                                             */
  float near_end_surface;  /* 0.98                                                          */
  float far_end_surface;   /* 1.02                                                          */
  float near_end;          /* 0.3                                                           */
  float sigmoid_coef;      /* 0.1                                                           */
  int min_nn_num;          /* 2                                                             */
  float w_color;
  int handle_dynamic;
  int use_color_in_tracking;
  const float* t_surface;  /* DEVICE [n_surface] torch.linspace(0,1,n)                      */
  const float* far;        /* DEVICE scalar min(5*mean(d), max(1.2*d)) (batch-global, Q9)   */
  const float* radius_query; /* DEVICE [R] per-ray dynamic query radius                     */
  const float* rand_feat;  /* DEVICE [32] feature of samples with < min_nn neighbours (Q6)
                              or NULL = zeros                                               */
  const float* rand_feat_color; /* the colour decoder's own draw (decoder_pointslam.py:463) */
} XrdPointCfg;

typedef struct {
  const float* geo_feats;      /* DEVICE [N][32]                                            */
  const uint8_t* frustum_mask; /* DEVICE [N] or NULL (multiplies geo_feats only, row P9)     */
  const float* col_feats;      /* DEVICE [N][32]; stage colour only                         */
} XrdPointFeats;

/* Colour decoder (slam/model_components/decoder_pointslam.py:313-542 MLP_color + :276-292
 * MLP_col_neighbor), all row-major [out][in] like nn.Linear:
 *   per neighbour k: f_k = nb_w2 . softplus100(nb_w1 . [sin, cos(2 pi (x_k - p) B_rel), col_feat_k]) ; c = sum_k w_k f_k
 *   h = softplus100(w[i] . h + b[i]) + (wc[i] . c + bc[i]),  i = 0..4, input cat after i = 2
 *   rgb = sigmoid(wo . h + bo);  first input = [sin, cos](2 pi p B). */
typedef struct {
  const float* B;      /* [3][20] fixed (GaussianFourierFeatureTransform, not learnable)   */
  const float* B_rel;  /* [3][10] learnable                                                */
  const float* nb_w1; const float* nb_b1; /* [128][52], [128]                              */
  const float* nb_w2; const float* nb_b2; /* [32][128], [32]                               */
  const float* w[5];  const float* b[5];  /* [128][40|128|128|168|128], [128]              */
  const float* wc[5]; const float* bc[5]; /* fc_c: [128][32], [128]                        */
  const float* wo;    const float* bo;    /* [3][128], [3]                                 */
} XrdPointColorDecoder;

/* Same shapes; every non-NULL array is ACCUMULATED into. */
typedef struct {
  float* B_rel;
  float* nb_w1; float* nb_b1; float* nb_w2; float* nb_b2;
  float* w[5]; float* b[5]; float* wc[5]; float* bc[5];
  float* wo; float* bo;
} XrdPointColorDecoderGrads;

typedef struct {
  float* rgb;              /* [R,3] (zeros in stage geometry)                               */
  float* depth;            /* [R]                                                           */
  float* uncertainty;      /* [R]                                                           */
  uint8_t* valid_ray_mask; /* [R]                                                           */
  float* z_vals;           /* [R,n_surface] optional                                        */
  float* losses;           /* [2] geo_loss, rgb_loss (already weighted)                     */
} XrdPointOut;

typedef struct {
  float* d_geo_feats;      /* [N][32] ACCUMULATED                                           */
  float* d_rays_o;         /* [R,3] or NULL                                                 */
  float* d_rays_d;
  float* d_col_feats;      /* [N][32] ACCUMULATED; stage colour, or NULL                    */
  XrdPointColorDecoderGrads* color; /* colour-decoder gradients or NULL (decoder fixed)     */
} XrdPointGrads;

/* Measurement / parity hook: arithmetic of the wide-MLP GEMMs (Point-SLAM colour stage and
 * the Vox-Fusion decoder):
 * 0 = fp32 SIMT, 1 = 3xTF32 tensor cores (default, fp32-level accuracy): wgmma / TMA
 * kernel where the shape qualifies, mma.sync otherwise, 2 = plain TF32 (mma.sync),
 * 3 = 3xTF32 on mma.sync only.  Thread-local, like the error state. */
int xrd_debug_gemm_mode(int mode);
/* bring-up hook of the wgmma GEMM (bit 0 swaps the descriptor strides); 0 = production */
int xrd_debug_gemm_variant(int variant);

/* The wide-MLP GEMM itself (unit tests): C[m][n] = act(sum_k A(m,k) B[k][n] + bias[m]) with
 * A(m,k) = transA ? A[k*lda+m] : A[m*lda+k]; act 0 none, 1 relu, 2 softplus(beta 100),
 * 3 sigmoid; result zeroed where relu_mask[m][n] <= 0; + addend[m][n].  DEVICE pointers. */
int xrd_debug_gemm(int M, int N, int K, const float* A, int lda, int transA, const float* B,
                   int ldb, float* C, int ldc, const float* bias, int act,
                   const float* relu_mask, int ldmask, const float* addend, int ldadd,
                   void* stream);

/* ... plus act_out[m][n] (the masked activation before the addend) and accumulate (C += ). */
int xrd_debug_gemm_ex(int M, int N, int K, const float* A, int lda, int transA, const float* B,
                      int ldb, float* C, int ldc, const float* bias, int act,
                      const float* relu_mask, int ldmask, const float* addend, int ldadd,
                      float* act_out, int ldact, int accumulate, void* stream);

/* The weight-gradient kernel of the per-point MLPs (unit tests): out[j][i] += sum_p B[j][p] A[i][p]
 * over P points (rows of Pp floats), B[j][p] dropped where bit (j & 31) of mask[j / 32][p] is
 * clear (mask may be NULL), bias[j] += sum_p B[j][p] (bias may be NULL).  DEVICE pointers. */
int xrd_debug_dw(int nA, int nB, int P, int Pp, const float* A, const float* B,
                 const uint32_t* mask, float* out, float* bias, void* stream);

size_t xrd_pointslam_workspace_bytes(int n_rays, int n_surface, int stage, int with_grads);

int xrd_pointslam_step(const XrdRays* rays, const XrdPointIndex* index,
                       const XrdPointFeats* feats, const XrdNiceDecoder* geo_decoder,
                       const XrdPointColorDecoder* color_decoder /* NULL in stage geometry */,
                       const XrdPointCfg* cfg, XrdPointOut* out, XrdPointGrads* grads,
                       void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* XRDSLAM_B200_H_ */
