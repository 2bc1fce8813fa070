"""Restatements of the camera-pose chain and the fused Adam step that a kernel can be held to
bit for bit or within a derived float64 bound.

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

  rays_fwd_f32      csrc/rays.cu k_fwd in numpy float32, in the kernel's operation order
                    ((d0 * M[c,0]) + (d1 * M[c,1])) + d2 * M[c,2]: every step is one correctly
                    rounded IEEE operation, so the kernel must agree bit for bit.
  rays_bwd_f64      csrc/rays.cu k_bwd in float64 plus the per-entry sum of |term| and the
                    per-pose ray count the summation-order-free bound needs.
  rodrigues_f64     csrc/pose.cu k_fwd / k_bwd (opt_pose.py's Rodrigues and what autograd
  rodrigues_bwd_f64 does through it) in float64, on the kernel's side of the theta <= 1e-8
                    identity branch.
  adam_f32          csrc/adam.cu upd / k_adam in numpy float32, in the kernel's operation order
                    (row mask, zero_grad, `dyn` scalars included): bit for bit.

numpy float32 arithmetic rounds every operation once and keeps subnormals, as the kernels do
(no --use_fast_math, no -ftz, no contraction into fma in these three expressions).
"""
from __future__ import annotations

import numpy as np

U32 = 2.0 ** -24                          # unit roundoff of float32
THETA_EPS = float(np.float32(1e-8))       # pose.cu: `th > 1e-8f`


def gamma(k):
    """gamma(k) = k u / (1 - k u), u = 2^-24: |fl(sum of k + 1 products) - exact| <= gamma(k)
    sum |terms| for ANY summation order (Higham, Accuracy and Stability, Lemma 3.1)."""
    k = np.asarray(k, np.float64)
    return k * U32 / (1.0 - k * U32)


def pose_rows(ids, R, n_poses):
    """-> (row [R] int64, live [R] bool): the pose row each ray reads (python negative indexing)
    and whether the id is in range (rays.cu pose_row)."""
    ids = np.zeros(R, np.int64) if ids is None else np.asarray(ids, np.int64)
    row = np.where(ids < 0, ids + n_poses, ids)
    live = (row >= 0) & (row < n_poses)
    return np.where(live, row, 0), live


# ------------------------------------------------------------------ rays ---
def rays_fwd_f32(dirs, ids, poses):
    """-> (rays_o, rays_d) [R,3] float32 of xrd_rays_from_poses; NaN for out-of-range ids."""
    dirs = np.asarray(dirs, np.float32)
    poses = np.asarray(poses, np.float32)
    row, live = pose_rows(ids, dirs.shape[0], poses.shape[0])
    M = poses[row]
    d0, d1, d2 = (dirs[:, j:j + 1] for j in range(3))
    rd = (d0 * M[:, :3, 0] + d1 * M[:, :3, 1]) + d2 * M[:, :3, 2]
    ro = M[:, :3, 3].copy()
    rd[~live] = np.nan
    ro[~live] = np.nan
    return ro, rd


def rays_bwd_f64(dirs, ids, n_poses, d_o, d_d):
    """-> (d_poses [n,4,4], abs_sum [n,4,4], n_p [n]) in float64 for xrd_rays_pose_grads:
    d_poses[p][c, j] = sum_r d_d[r, c] dirs[r, j], d_poses[p][c, 3] = sum_r d_o[r, c] over the
    in-range rays r of pose p (either gradient may be None); abs_sum is the same sum of |term|,
    n_p the number of rays of pose p.  The bottom row stays 0.  fp32 forms each term with at
    most one rounding and adds n_p of them, so |kernel - d_poses| <= gamma(n_p + 2) abs_sum."""
    dirs = np.asarray(dirs, np.float64)
    R = dirs.shape[0]
    row, live = pose_rows(ids, R, n_poses)
    t = np.zeros((R, 4, 4))
    if d_d is not None:
        t[:, :3, :3] = np.asarray(d_d, np.float64)[:, :, None] * dirs[:, None, :]
    if d_o is not None:
        t[:, :3, 3] = np.asarray(d_o, np.float64)
    t[~live] = 0.0
    d_poses, abs_sum = np.zeros((n_poses, 4, 4)), np.zeros((n_poses, 4, 4))
    np.add.at(d_poses, row[live], t[live])
    np.add.at(abs_sum, row[live], np.abs(t[live]))
    n_p = np.bincount(row[live], minlength=n_poses)
    return d_poses, abs_sum, n_p


# ------------------------------------------------------------------ poses ---
def _skew(k):
    z = np.zeros(k.shape[:-1])
    return np.stack([np.stack([z, -k[..., 2], k[..., 1]], -1),
                     np.stack([k[..., 2], z, -k[..., 0]], -1),
                     np.stack([-k[..., 1], k[..., 0], z], -1)], -2)


def _axis(rot, thresh):
    w = np.asarray(rot, np.float64)
    th = np.linalg.norm(w, axis=-1)
    on = th > thresh
    k = w / np.where(on, th, 1.0)[:, None]
    return th, on, k


def rodrigues_f64(rot, trans):
    """-> c2w [n,4,4] float64: R = I + sin(th) K + (1 - cos(th)) K^2, K = skew(w / th), and
    R = I where th <= 1e-8 (pose.cu k_fwd, opt_pose.py axis_angle_to_rotation_matrix)."""
    th, on, k = _axis(rot, THETA_EPS)
    K = _skew(k)
    n = th.shape[0]
    c1 = 2 * np.sin(th / 2) ** 2  # = 1 - cos(th) without the cancellation at small th
    R = np.eye(3) + np.sin(th)[:, None, None] * K + c1[:, None, None] * (K @ K)
    R[~on] = np.eye(3)
    M = np.zeros((n, 4, 4))
    M[:, :3, :3] = R
    M[:, :3, 3] = np.asarray(trans, np.float64)
    M[:, 3, 3] = 1.0
    return M


def rodrigues_bwd_f64(rot, d_c2w, fixed=None, thresh=THETA_EPS, project=True, transpose_k=True):
    """-> (d_rot [n,3], d_trans [n,3]) float64, the chain of G = d_c2w through rodrigues_f64
    (pose.cu k_bwd's header comment):
        dL/dK = s G + c1 (G K^T + K^T G),  dL/dk from the skew layout,
        dL/dth = cos(th) <G,K> + sin(th) <G,K^2>,
        dL/dw = (dL/dk - (dL/dk . k) k) / th + dL/dth k.
    d_trans = G[:3, 3]; rows with th <= thresh get no rotation gradient, fixed rows nothing.
    thresh / project / transpose_k other than the defaults are the mutation tests' faults (the
    threshold moved, the projection dropped, K instead of K^T in dL/dK)."""
    G4 = np.asarray(d_c2w, np.float64)
    th, on, k = _axis(rot, thresh)
    G = G4[:, :3, :3]
    K = _skew(k)
    K2 = K @ K
    Kt = np.swapaxes(K, -1, -2) if transpose_k else K
    s = np.sin(th)[:, None, None]
    dK = s * G + 2 * np.sin(th / 2)[:, None, None] ** 2 * (G @ Kt + Kt @ G)
    dk = np.stack([dK[:, 2, 1] - dK[:, 1, 2], dK[:, 0, 2] - dK[:, 2, 0],
                   dK[:, 1, 0] - dK[:, 0, 1]], -1)
    dth = np.cos(th) * (G * K).sum((1, 2)) + np.sin(th) * (G * K2).sum((1, 2))
    dot = (dk * k).sum(-1, keepdims=True) if project else 0.0
    d_rot = (dk - dot * k) / np.where(on, th, 1.0)[:, None] + dth[:, None] * k
    d_rot[~on] = 0.0
    d_trans = G4[:, :3, 3].copy()
    if fixed is not None:
        fx = np.asarray(fixed).astype(bool)
        d_rot[fx] = 0.0
        d_trans[fx] = 0.0
    return d_rot, d_trans


# ------------------------------------------------------------------ Adam ---
def adam_f32(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay,
             bias_correction1, bias_correction2, row_mask=None, row_len=1, zero_grad=0,
             dyn=None):
    """One xrd_adam_step on one tensor in numpy float32 -> (param, grad, exp_avg, exp_avg_sq)
    after the call.  Scalars enter as the float32 fields of XrdAdamTensor; `dyn` = (lr, bc1, bc2)
    overrides the host values.  Rows whose row_mask entry is 0 keep param and both moments;
    zero_grad != 0 clears every gradient, masked rows included."""
    f = np.float32
    p = np.array(param, f).reshape(-1)
    g = np.array(grad, f).reshape(-1)
    m = np.array(exp_avg, f).reshape(-1)
    v = np.array(exp_avg_sq, f).reshape(-1)
    lr, bc1, bc2 = (f(x) for x in (dyn if dyn is not None else
                                   (lr, bias_correction1, bias_correction2)))
    b1, b2, eps, wd = f(beta1), f(beta2), f(eps), f(weight_decay)
    step_size = lr / bc1
    inv_sqrt_bc2 = f(1) / np.sqrt(bc2)
    live = np.ones(p.shape, bool) if row_mask is None else \
        np.repeat(np.asarray(row_mask).astype(bool), row_len)[:p.size]
    pp, gg, mm, vv = p[live], g[live], m[live], v[live]
    if wd != 0:
        gg = gg + wd * pp
    mm = mm + (gg - mm) * (f(1) - b1)
    vv = vv * b2 + ((f(1) - b2) * gg) * gg
    denom = np.sqrt(vv) * inv_sqrt_bc2 + eps
    pp = pp - step_size * (mm / denom)
    p[live], m[live], v[live] = pp, mm, vv
    if zero_grad:
        g[:] = 0
    return p, g, m, v


def adam_f64(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay,
             bias_correction1, bias_correction2):
    """The same rule in float64 (no mask) on the float32 values of the scalars, 1 - beta1 and
    1 - beta2 included: the rounding-free value adam_f32 approximates."""
    lr, beta1, beta2, eps, weight_decay, bias_correction1, bias_correction2 = (
        float(np.float32(x)) for x in (lr, beta1, beta2, eps, weight_decay, bias_correction1,
                                       bias_correction2))
    p, g, m, v = (np.array(x, np.float64).reshape(-1) for x in (param, grad, exp_avg, exp_avg_sq))
    if weight_decay != 0:
        g = g + weight_decay * p
    m = m + (g - m) * (1 - beta1)
    v = v * beta2 + (1 - beta2) * g * g
    p = p - lr / bias_correction1 * m / (np.sqrt(v) / np.sqrt(bias_correction2) + eps)
    return p, m, v
