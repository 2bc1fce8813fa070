"""ds-eval's reconstruction metrics (scripts/utils/eval_recon.py, evaluate_3d_reconstruction,
reference @ f0366f20) restated twice.

(a) numpy in csrc/eval.cu's exact order (semantics in include/xrdslam_b200.h, xrd_eval_* /
    xrd_nn_*): the chunked float64 area prefix and both samplers with the uniforms given, an
    fp32 brute-force nearest neighbour with the kernel's formula and tie rule, the chunked
    float64 reductions, the ICP loop and the metric assembly.  The CUDA path matches it bit for
    bit (tests/test_eval_recon_gpu.py).
(b) ``ckdtree_dist``: the reference's own arithmetic, scipy's cKDTree in float64, the tool
    calc_3d_metric uses.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
AREA_CHUNK = 256     # XRD_EVAL_AREA_CHUNK
RED_CHUNK = 4096     # XRD_EVAL_RED_CHUNK
RED_THREADS = 256


# ---------------------------------------------------------------- sampling ---
def area_prefix(verts, faces):
    """-> (cum f64 [F], total f64): sequential inside chunks of AREA_CHUNK faces, plus the
    chunk's offset (sequential sum of the earlier chunk totals)."""
    V = np.asarray(verts, f32).astype(np.float64)
    F = np.asarray(faces, np.int64)
    a = V[F[:, 0]]
    e1, e2 = V[F[:, 1]] - a, V[F[:, 2]] - a
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    area = 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)
    n = area.shape[0]
    nc = -(-n // AREA_CHUNK)
    pad = np.zeros(nc * AREA_CHUNK)
    pad[:n] = area
    local = np.cumsum(pad.reshape(nc, AREA_CHUNK), axis=1)
    tot = local[:, -1]
    off = np.concatenate([[0.0], np.cumsum(tot)[:-1]])
    cum = (off[:, None] + local).reshape(-1)[:n]
    return cum, float(np.cumsum(tot)[-1])


def sample_trimesh(verts, faces, U):
    """trimesh sample_surface with uniforms U f32 [n,3] -> (points f32 [n,3], face ids)."""
    V = np.asarray(verts, f32)
    F = np.asarray(faces, np.int64)
    U = np.asarray(U, f32)
    cum, total = area_prefix(V, F)
    fi = np.minimum(np.searchsorted(cum, U[:, 0].astype(np.float64) * total, side='left'),
                    len(F) - 1)
    a, b = U[:, 1].copy(), U[:, 2].copy()
    fold = (a + b) > f32(1)
    a[fold] = np.abs(a[fold] - f32(1))
    b[fold] = np.abs(b[fold] - f32(1))
    p0, p1, p2 = V[F[fi, 0]], V[F[fi, 1]], V[F[fi, 2]]
    return p0 + (a[:, None] * (p1 - p0) + b[:, None] * (p2 - p0)), fi


def sample_open3d(verts, faces, n, U):
    """open3d sample_points_uniformly(n) with uniforms U f32 [n,2] -> (points, face ids)."""
    V = np.asarray(verts, f32)
    F = np.asarray(faces, np.int64)
    U = np.asarray(U, f32)
    cum, total = area_prefix(V, F)
    ends = _round_half_away((cum / total) * float(n))
    fi = np.minimum(np.searchsorted(ends, np.arange(n, dtype=np.float64), side='right'),
                    len(F) - 1)
    s = np.sqrt(U[:, 0])
    w0 = f32(1) - s
    w1 = s * (f32(1) - U[:, 1])
    w2 = s * U[:, 1]
    p0, p1, p2 = V[F[fi, 0]], V[F[fi, 1]], V[F[fi, 2]]
    return (w0[:, None] * p0 + w1[:, None] * p1) + w2[:, None] * p2, fi


def _round_half_away(x):
    """C's round() for x >= 0 (x - floor(x) is exact)."""
    fl = np.floor(x)
    return np.where(x - fl >= 0.5, fl + 1.0, fl)


# ---------------------------------------------------------------- nearest neighbour ---
def nn_brute(queries, targets, radius=None, chunk=256):
    """Nearest target per query, fp32 d2 = (dx*dx + dy*dy) + dz*dz with dx = q - p, ties to the
    smallest id.  radius: only d2 <= f32(r) * f32(r); none -> (inf, -1).  -> (dist f32, ids)."""
    Q = np.asarray(queries, f32).reshape(-1, 3)
    P = np.asarray(targets, f32).reshape(-1, 3)
    dist = np.empty(len(Q), f32)
    ids = np.empty(len(Q), np.int32)
    r2 = None if radius is None or not radius > 0 or not np.isfinite(radius) else \
        f32(radius) * f32(radius)
    for s in range(0, len(Q), chunk):
        q = Q[s:s + chunk]
        dx = q[:, None, 0] - P[None, :, 0]
        dy = q[:, None, 1] - P[None, :, 1]
        dz = q[:, None, 2] - P[None, :, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        j = np.argmin(d2, axis=1)          # first minimum: the smallest id
        b = d2[np.arange(len(q)), j]
        ok = np.ones(len(q), bool) if r2 is None else b <= r2
        dist[s:s + chunk] = np.where(ok, np.sqrt(b), np.inf)
        ids[s:s + chunk] = np.where(ok, j, -1)
    return dist, ids


def ckdtree_dist(queries, targets):
    """The reference's distances: scipy cKDTree(targets).query(queries) in float64."""
    from scipy.spatial import cKDTree
    d, i = cKDTree(np.asarray(targets, np.float64)).query(np.asarray(queries, np.float64))
    return d, i


# ---------------------------------------------------------------- reductions ---
def reduce_f64(vals):
    """Sum of the rows of vals f64 [n, K] in xrd_eval_*_stats' order -> f64 [K]."""
    vals = np.asarray(vals, np.float64)
    n, K = vals.shape
    npart = max(1, -(-n // RED_CHUNK))
    pad = np.zeros((npart * RED_CHUNK, K))
    pad[:n] = vals
    v = pad.reshape(npart, RED_CHUNK // RED_THREADS, RED_THREADS, K)
    acc = np.zeros((npart, RED_THREADS, K))
    for m in range(RED_CHUNK // RED_THREADS):
        acc = acc + v[:, m]
    s = RED_THREADS // 2
    while s > 0:
        acc[:, :s] = acc[:, :s] + acc[:, s:2 * s]
        s //= 2
    part = acc[:, 0]
    out = np.zeros(K)
    for p in range(npart):
        out = out + part[p]
    return out


def dist_stats(d, tau):
    """(sum d, sum d*d, count of d < tau in fp32) as f64 [3]."""
    d = np.asarray(d, f32)
    x = d.astype(np.float64)
    return reduce_f64(np.stack([x, x * x, (d < f32(tau)).astype(np.float64)], 1))


def icp_stats(src, tgt, ids, d):
    """(count, sum s, sum t, sum s t^T row-major, sum d*d) over ids >= 0, f64 [17]."""
    src = np.asarray(src, f32).astype(np.float64)
    tgt = np.asarray(tgt, f32).astype(np.float64)
    ids = np.asarray(ids)
    m = ids >= 0
    t = np.zeros_like(src)
    t[m] = tgt[ids[m]]
    s = np.where(m[:, None], src, 0.0)
    x = np.where(m, np.asarray(d, f32).astype(np.float64), 0.0)
    st = (s[:, :, None] * t[:, None, :]).reshape(-1, 9)
    return reduce_f64(np.concatenate([m[:, None].astype(np.float64), s, t, st, (x * x)[:, None]],
                                     1))


def transform(points, T):
    """fp32(((T0 x + T1 y) + T2 z) + T3) per row, f64 arithmetic."""
    p = np.asarray(points, f32).astype(np.float64)
    T = np.asarray(T, np.float64)
    out = ((T[None, :3, 0] * p[:, :1] + T[None, :3, 1] * p[:, 1:2]) + T[None, :3, 2] * p[:, 2:3]) \
        + T[None, :3, 3]
    return out.astype(f32)


# ---------------------------------------------------------------- ICP ---
def umeyama(stats):
    """Rigid (no scale) Umeyama from icp_stats -> 4x4 f64 (identity without correspondences)."""
    n = stats[0]
    T = np.eye(4)
    if n <= 0:
        return T
    mu_s, mu_t = stats[1:4] / n, stats[4:7] / n
    sig = stats[7:16].reshape(3, 3).T / n - np.outer(mu_t, mu_s)
    U, _, Vt = np.linalg.svd(sig)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    T[:3, :3] = R
    T[:3, 3] = mu_t - R @ mu_s
    return T


def fitness_rmse(stats, n_src):
    c = stats[0]
    return (c / n_src if n_src else 0.0), (float(np.sqrt(stats[16] / c)) if c else 0.0)


def registration_icp(src, tgt, max_correspondence_distance, init=None, max_iteration=30,
                     relative_fitness=1e-6, relative_rmse=1e-6, nn=None):
    """open3d's point-to-point ICP (from memory, unverified) with every transform applied to the
    original source once -> dict(transformation, fitness, inlier_rmse, iterations)."""
    nn = nn_brute if nn is None else nn
    src = np.asarray(src, f32)
    T = np.eye(4) if init is None else np.asarray(init, np.float64)

    def corr(T):
        s = transform(src, T)
        d, ids = nn(s, tgt, max_correspondence_distance)
        return icp_stats(s, tgt, ids, d)

    st = corr(T)
    fit, rmse = fitness_rmse(st, len(src))
    it = 0
    for it in range(1, max_iteration + 1):
        T = umeyama(st) @ T
        st = corr(T)
        f2, r2 = fitness_rmse(st, len(src))
        done = abs(fit - f2) < relative_fitness and abs(rmse - r2) < relative_rmse
        fit, rmse = f2, r2
        if done:
            break
    return dict(transformation=T, fitness=fit, inlier_rmse=rmse, iterations=it)


# ---------------------------------------------------------------- metrics ---
def fscore_assembly(d1, d2, tau):
    """get_f1_score_histo's precision / recall / F (F = 0 when both are 0) and the statistics
    EvaluateHisto writes, from the float64 reductions."""
    s1, s2 = dist_stats(d1, tau), dist_stats(d2, tau)
    n1, n2 = len(d1), len(d2)
    p, r = s1[2] / n1, s2[2] / n2
    f = 2 * r * p / (r + p) if r + p > 0 else 0.0
    return dict(precision=p, recall=r, fscore=f, mean1=s1[0] / n1, mean2=s2[0] / n2)


def calc_3d_from_points(rec_pts, gt_pts):
    """accuracy / completion (cm) and the 5 cm completion ratio (%) of two point sets."""
    d_rg, _ = nn_brute(rec_pts, gt_pts)
    d_gr, _ = nn_brute(gt_pts, rec_pts)
    a = dist_stats(d_rg, 0.05)
    c = dist_stats(d_gr, 0.05)
    return {'accuracy': a[0] / len(d_rg) * 100, 'completion': c[0] / len(d_gr) * 100,
            'completion ratio': c[2] / len(d_gr) * 100}


def nn_kdtree_f32(queries, targets, radius=None, k=8):
    """nn_brute's answer (fp32 d2, ties to the smallest id) from the k nearest candidates of a
    float64 cKDTree: for meshes too large for the brute force."""
    from scipy.spatial import cKDTree
    Q = np.asarray(queries, f32).reshape(-1, 3)
    P = np.asarray(targets, f32).reshape(-1, 3)
    k = min(k, len(P))
    _, cand = cKDTree(P.astype(np.float64)).query(Q.astype(np.float64), k=k)
    cand = cand.reshape(len(Q), k)
    dx = Q[:, None, 0] - P[cand, 0]
    dy = Q[:, None, 1] - P[cand, 1]
    dz = Q[:, None, 2] - P[cand, 2]
    d2 = (dx * dx + dy * dy) + dz * dz
    order = np.lexsort((cand, d2), axis=1)[:, 0]
    j = cand[np.arange(len(Q)), order]
    b = d2[np.arange(len(Q)), order]
    ok = np.ones(len(Q), bool)
    if radius is not None and radius > 0 and np.isfinite(radius):
        ok = b <= f32(radius) * f32(radius)
    return np.where(ok, np.sqrt(b), np.inf).astype(f32), np.where(ok, j, -1).astype(np.int32)


def philox_uniforms(seed, n, per):
    """common.cuh philox4(seed, k) for k < n, first `per` values -> f32 [n, per]."""
    M = np.uint64(0xFFFFFFFF)
    idx = np.arange(n, dtype=np.uint64)
    c = [idx & M, idx >> np.uint64(32), np.zeros(n, np.uint64), np.zeros(n, np.uint64)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & M
        hi1, lo1 = p1 >> np.uint64(32), p1 & M
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M
        k1 = (k1 + np.uint64(0xBB67AE85)) & M
    s = f32(2.3283064365386963e-10)
    out = [((x.astype(np.uint32).astype(f32) + f32(0.5)) * s) * f32(0.99999994) for x in c[:per]]
    return np.stack(out, 1)


def ds_eval_3d(rec_v, rec_f, gt_v, gt_f, transform_matrix, seed=0, tau=0.01,
               n_samples=200000, nn=nn_kdtree_f32):
    """eval.EvalMatrics' reconstruction half in this restatement: the given transform, a
    30-iteration ICP, both metrics on Philox draws (seeds seed, seed + 1 for calc_3d_metric and
    seed + 2 for run_evaluation) -> the merged dict."""
    rec_v, gt_v = np.asarray(rec_v, f32), np.asarray(gt_v, f32)
    T0 = np.asarray(transform_matrix, np.float64)
    res = {}
    for pass_seed, fscore in ((seed, False), (seed + 2, True)):
        icp = registration_icp(transform(rec_v, T0), gt_v, 0.1, max_iteration=30, nn=nn)
        rv = transform(rec_v, icp['transformation'] @ T0)
        if not fscore:
            rp, _ = sample_trimesh(rv, rec_f, philox_uniforms(pass_seed, n_samples, 3))
            gp, _ = sample_trimesh(gt_v, gt_f, philox_uniforms(pass_seed + 1, n_samples, 3))
            d_rg, _ = nn(rp, gp)
            d_gr, _ = nn(gp, rp)
            a, c = dist_stats(d_rg, 0.05), dist_stats(d_gr, 0.05)
            res.update({'accuracy': a[0] / n_samples * 100,
                        'completion': c[0] / n_samples * 100,
                        'completion ratio': c[2] / n_samples * 100})
            continue
        if len(gt_v) < len(rv):
            gp, _ = sample_open3d(gt_v, gt_f, len(rv), philox_uniforms(pass_seed, len(rv), 2))
            d1, _ = nn(rv, gp)
            d2, _ = nn(gt_v, rv)
        else:
            rp, _ = sample_open3d(rv, rec_f, len(gt_v), philox_uniforms(pass_seed, len(gt_v), 2))
            d1, _ = nn(rv, gt_v)
            d2, _ = nn(gt_v, rp)
        h = fscore_assembly(d1, d2, tau)
        res.update({'dist_threshold': tau, 'precision': h['precision'], 'recall': h['recall'],
                    'f-score': h['fscore'], 'mean precision': h['mean1'],
                    'mean recall': h['mean2']})
    return res
