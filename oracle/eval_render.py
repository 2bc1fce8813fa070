"""numpy restatement of csrc/eval_render.cu in the kernels' arithmetic (test infrastructure
only, never on the product path): the depth rasteriser (clip, snap, int64 edge functions, f64
plane depth), check_proj, the per-view depth-L1 sums and the sequential view-sampler loop of
calc_2d_metric (scripts/utils/eval_recon.py:212-232, reference @ f0366f20).

numpy's float64 / float32 elementwise operations round to nearest and are never contracted, so
writing the kernels' expressions in the same order reproduces them bit for bit."""
from __future__ import annotations

import numpy as np

SUB = 256          # XRD_EVAL_RENDER_SUBPIXEL
GUARD = 2097152.0  # XRD_EVAL_RENDER_GUARD
f32 = np.float32


def to_cam(M, w):
    """M f64 [3,4], w f64 [..., 3] -> camera-space f64 [..., 3], ((r0 x + r1 y) + r2 z) + t."""
    x, y, z = w[..., 0], w[..., 1], w[..., 2]
    return np.stack([((M[a, 0] * x + M[a, 1] * y) + M[a, 2] * z) + M[a, 3] for a in range(3)], -1)


def plane_d(cam, k, p):
    x, y, z = p
    if k == 0:
        return z - cam['near']
    if k == 1:
        return GUARD * z - cam['fx'] * x
    if k == 2:
        return GUARD * z + cam['fx'] * x
    if k == 3:
        return GUARD * z - cam['fy'] * y
    return GUARD * z + cam['fy'] * y


def _cross_point(cam, k, a, b):
    if tuple(b) < tuple(a):
        a, b = b, a
    da, db = plane_d(cam, k, a), plane_d(cam, k, b)
    t = da / (da - db)
    return tuple(a[i] + t * (b[i] - a[i]) for i in range(3))


def clip_poly(cam, P):
    """Sutherland-Hodgman against near, then the four guard planes; P a list of (x, y, z)."""
    for k in range(5):
        if not P:
            break
        Q = []
        n = len(P)
        for i in range(n):
            cur, prev = P[i], P[i - 1]
            ci, pi = plane_d(cam, k, cur) >= 0.0, plane_d(cam, k, prev) >= 0.0
            if ci:
                if not pi:
                    Q.append(_cross_point(cam, k, prev, cur))
                Q.append(cur)
            elif pi:
                Q.append(_cross_point(cam, k, prev, cur))
        P = Q if len(Q) >= 3 else []
    return P


def _inside_all(cam, p):
    return all(plane_d(cam, k, p) >= 0.0 for k in range(5))


def _plane(cam, p0, p1, p2):
    e1 = [p1[i] - p0[i] for i in range(3)]
    e2 = [p2[i] - p0[i] for i in range(3)]
    nx = e1[1] * e2[2] - e1[2] * e2[1]
    ny = e1[2] * e2[0] - e1[0] * e2[2]
    nz = e1[0] * e2[1] - e1[1] * e2[0]
    k = (nx * p0[0] + ny * p0[1]) + nz * p0[2]
    ax, ay = nx / cam['fx'], ny / cam['fy']
    c0 = nz - (ax * cam['cx'] + ay * cam['cy'])
    return ax, ay, c0, k


def _snap(v):
    return np.int64(np.rint(np.float64(v) * SUB))


def _project(cam, p):
    u = (cam['fx'] * p[0]) / p[2] + cam['cx']
    v = (cam['fy'] * p[1]) / p[2] + cam['cy']
    return _snap(u), _snap(v)


def _raster_tri(cam, a, b, d, pl, img):
    X, Y = zip(*(_project(cam, p) for p in (a, b, d)))
    X, Y = np.array(X, np.int64), np.array(Y, np.int64)
    x0 = max(0, int((X.min() + SUB - 1) >> 8))
    x1 = min(cam['W'] - 1, int(X.max() >> 8))
    y0 = max(0, int((Y.min() + SUB - 1) >> 8))
    y1 = min(cam['H'] - 1, int(Y.max() >> 8))
    if x0 > x1 or y0 > y1:
        return
    area = (X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0])
    if area == 0:
        return
    jj, ii = np.meshgrid(np.arange(y0, y1 + 1, dtype=np.int64),
                         np.arange(x0, x1 + 1, dtype=np.int64), indexing='ij')
    px, py = ii << 8, jj << 8
    w0 = (X[2] - X[1]) * (py - Y[1]) - (Y[2] - Y[1]) * (px - X[1])
    w1 = (X[0] - X[2]) * (py - Y[2]) - (Y[0] - Y[2]) * (px - X[2])
    w2 = (X[1] - X[0]) * (py - Y[0]) - (Y[1] - Y[0]) * (px - X[0])
    cov = ((w0 >= 0) & (w1 >= 0) & (w2 >= 0)) if area > 0 else ((w0 <= 0) & (w1 <= 0) & (w2 <= 0))
    if not cov.any():
        return
    ax, ay, c0, k = pl
    ic, jc = ii[cov].astype(np.float64), jj[cov].astype(np.float64)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        z = (k / ((ax * ic + ay * jc) + c0)).astype(f32)
    keep = (z > 0) & (z <= f32(cam['far'])) & np.isfinite(z)
    jk, ik, zk = jj[cov][keep], ii[cov][keep], z[keep]
    cur = img[jk, ik]
    img[jk, ik] = np.where((cur == 0) | (zk < cur), zk, cur)


def render_depth(verts, faces, w2c, cam):
    """verts f32 [V,3], faces i32 [F,3], w2c f64 [n,3,4], cam dict(H, W, fx, fy, cx, cy, near,
    far) -> depth f32 [n,H,W] (0 = nothing drawn), as xrd_eval_render_depth."""
    V = np.asarray(verts, f32).astype(np.float64)
    F = np.asarray(faces, np.int64)
    w2c = np.asarray(w2c, np.float64).reshape(-1, 3, 4)
    out = np.zeros((len(w2c), cam['H'], cam['W']), f32)
    W3 = V[F]  # [F, 3 corners, 3]
    for b, M in enumerate(w2c):
        Pc = to_cam(M, W3)  # [F, 3, 3]
        live = ~(Pc[:, :, 2] < cam['near']).all(1)
        for f in np.nonzero(live)[0]:
            P = [tuple(float(c) for c in Pc[f, k]) for k in range(3)]
            pl = _plane(cam, *P)
            if pl[3] == 0.0:
                continue
            if not all(_inside_all(cam, p) for p in P):
                P = clip_poly(cam, P)
            for t in range(1, len(P) - 1):
                _raster_tri(cam, P[0], P[t], P[t + 1], pl, out[b])
    return out


# ---------------------------------------------------------------- check_proj ---
def seen_w2c(c2w):
    """check_proj's w2c: columns 1 and 2 of c2w negated, inverted in f64, then fp32 rows 0..2."""
    c = np.array(c2w, np.float64, copy=True)
    c[..., :3, 1] *= -1.0
    c[..., :3, 2] *= -1.0
    return np.linalg.inv(c).astype(f32)[..., :3, :4]


def check_proj(points, W, H, fx, fy, cx, cy, c2w):
    """xrd_eval_points_seen for one view, in fp32 numpy."""
    m = seen_w2c(c2w)
    p = np.asarray(points, f32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    c = [((m[a, 0] * x + m[a, 1] * y) + m[a, 2] * z) + m[a, 3] for a in range(3)]
    xn = -c[0]
    zz = c[2] + f32(1e-5)
    with np.errstate(divide='ignore', invalid='ignore'):
        u = (f32(fx) * xn + f32(cx) * c[2]) / zz
        v = (f32(fy) * c[1] + f32(cy) * c[2]) / zz
    mask = (f32(0) <= -zz) & (u < f32(W)) & (u > 0) & (v < f32(H)) & (v > 0)
    return bool(mask.any())


# ---------------------------------------------------------------- sums and sampler ---
def depth_l1_sums(gt, rec):
    """xrd_eval_depth_l1: f64 [n,2] = (sum |gt - rec|, count) over rec > 0, thread-strided in
    256 lanes then the fixed tree."""
    gt = np.asarray(gt, f32).reshape(len(gt), -1)
    rec = np.asarray(rec, f32).reshape(len(rec), -1)
    out = np.zeros((len(gt), 2))
    for b in range(len(gt)):
        n = gt.shape[1]
        pad = (-n) % 256
        g = np.concatenate([gt[b], np.zeros(pad, f32)]).reshape(-1, 256)
        r = np.concatenate([rec[b], np.zeros(pad, f32)]).reshape(-1, 256)
        ok = r > 0
        d = np.where(ok, np.abs(g - r).astype(np.float64), 0.0)
        s, c = np.zeros(256), np.zeros(256)
        for row in range(len(d)):  # each lane in pixel order
            s = np.where(ok[row], s + d[row], s)
            c = np.where(ok[row], c + 1.0, c)
        h = 128
        while h:
            s = s[:h] + s[h:2 * h]
            c = c[:h] + c[h:2 * h]
            h >>= 1
        out[b] = s[0], c[0]
    return out


def sample_views_sequential(pc_unseen, extents, transform, n_imgs, seed, W=500, H=500, fx=300.,
                            fy=300., cx=249.5, cy=249.5, max_candidates=None):
    """calc_2d_metric's view loop, one candidate at a time (eval_recon.py:212-232), with seeded
    random.Random / numpy RandomState instances -> c2w f64 [n_imgs,4,4]."""
    import random

    from xrdslam_b200.eval_recon import volume_rectangular, viewmatrix
    pyr, npr = random.Random(seed), np.random.RandomState(seed)
    views, tried = [], 0
    limit = max_candidates or 1000 * n_imgs
    for _ in range(n_imgs):
        while True:
            if tried >= limit:
                raise RuntimeError('no view')
            tried += 1
            origin = volume_rectangular(extents, 1, transform, npr).reshape(-1)
            target = [round(pyr.uniform(-10000, +10000), 2) for _ in range(3)]
            target = np.array(target) - np.array(origin)
            c2w = np.eye(4)
            c2w[:3, :] = viewmatrix(target, [0, 0, -1], origin)
            if not check_proj(pc_unseen, W, H, fx, fy, cx, cy, c2w):
                break
        views.append(c2w)
    return np.array(views)
