"""ds-eval's 3D reconstruction metrics on the device (scripts/utils/eval_recon.py and
third_party/evaluate_3d_reconstruction_lib, reference @ f0366f20), on csrc/eval.cu.

The reference needs open3d (ICP, sample_points_uniformly, compute_point_cloud_distance),
trimesh (sample_surface) and scipy's cKDTree.  Here surface sampling, the exact nearest-neighbour
distances, ICP's correspondences and sums, and the means / counts run in CUDA; medians and
histograms use torch on the device, and each ICP iteration reads 17 doubles back for the 3x3
SVD.  Semantics are written down in include/xrdslam_b200.h (xrd_eval_*, xrd_nn_*).  The draws
are Philox (seeded), the reference's are unseeded: the metrics are statistically equivalent to
the reference's, not equal.  Names, signatures and dict keys follow the reference.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _cabi
from ._cabi import XRD_EVAL_OPEN3D, XRD_EVAL_TRIMESH, XrdNnIndex, check, ptr

N_SAMPLES = 200000      # calc_3d_metric's sample_surface count
ICP_THRESHOLD = 0.1     # max_correspondence_distance of every ICP in ds-eval
PLOT_STRETCH = 5


def _device(device=None):
    dev = torch.device(device if device is not None else 'cuda:0')
    if dev.type != 'cuda':
        raise RuntimeError('xrdslam_b200 has no CPU path: the reconstruction metrics run on a '
                           'CUDA device')
    return dev


def _pts(x, dev):
    t = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float32)))
    return t.to(dev, torch.float32).reshape(-1, 3).contiguous()


def load_mesh(mesh):
    """A PLY path, a TriMesh-like object (vertices, faces) or a (vertices, faces) pair ->
    (vertices, faces or None)."""
    if isinstance(mesh, (str, os.PathLike)):
        from .io_formats import read_ply
        v, f, _ = read_ply(str(mesh))
        return v, f
    if hasattr(mesh, 'vertices'):
        return mesh.vertices, getattr(mesh, 'faces', None)
    if isinstance(mesh, (tuple, list)) and len(mesh) == 2:
        return mesh[0], mesh[1]
    return mesh, None


# ---------------------------------------------------------------- kernels ---
def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def sample_surface(verts, faces, n, mode, uniforms=None, seed=0, device=None):
    """Area-weighted samples on a triangle mesh: mode XRD_EVAL_TRIMESH (trimesh sample_surface)
    or XRD_EVAL_OPEN3D (open3d sample_points_uniformly).  uniforms DEVICE f32 [n,3] / [n,2] or
    None (Philox with `seed`).  -> (points f32 [n,3], face ids i32 [n]) on the device.  A mesh
    without faces or area, with a face index outside [0, V) or a non-finite vertex raises."""
    dev = _device(device)
    v = _pts(verts, dev)
    if faces is None:
        faces = np.zeros((0, 3), np.int32)
    f = (faces if torch.is_tensor(faces) else torch.from_numpy(np.asarray(faces, np.int32))
         ).to(dev, torch.int32).reshape(-1, 3).contiguous()
    lib = _cabi.lib()
    nF = f.shape[0]
    nb = lib.xrd_eval_surface_workspace_bytes(nF)
    ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
    cum = torch.empty(max(nF, 1), dtype=torch.float64, device=dev)
    total = torch.empty(1, dtype=torch.float64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    fid = torch.empty(n, dtype=torch.int32, device=dev)
    if uniforms is not None:
        uniforms = uniforms.to(dev, torch.float32).contiguous()
        if uniforms.shape != (n, 3 if mode == XRD_EVAL_TRIMESH else 2):
            raise ValueError(f'uniforms must be [{n}, {3 if mode == XRD_EVAL_TRIMESH else 2}]')
    with torch.cuda.device(dev):
        s = _stream(dev)
        check('xrd_eval_surface_prepare', lib.xrd_eval_surface_prepare(
            ptr(v), v.shape[0], ptr(f), nF, ptr(cum), ptr(total), ptr(status), ptr(ws), nb, s))
        check('xrd_eval_sample_surface', lib.xrd_eval_sample_surface(
            ptr(v), ptr(f), nF, ptr(cum), ptr(total), ptr(status), mode, n, ptr(uniforms),
            seed, ptr(out), ptr(fid), s))
        check('xrd_eval_surface_prepare', int(status.item()))
    return out, fid


class NNIndex:
    """Exact nearest-neighbour index over DEVICE target points (xrd_nn_*): the box is read once
    on the host, the rest is built on the device."""

    def __init__(self, targets, device=None):
        dev = _device(device) if not torch.is_tensor(targets) or not targets.is_cuda else \
            targets.device
        self.points = _pts(targets, dev)
        self.device = dev
        n = self.points.shape[0]
        if n < 1:
            raise ValueError('the nearest-neighbour index needs at least one target point')
        lo, hi = torch.aminmax(self.points, dim=0)
        box = torch.stack([lo, hi]).double().cpu().numpy()
        lib = _cabi.lib()
        I = XrdNnIndex()
        check('xrd_nn_layout', lib.xrd_nn_layout(
            n, (C.c_double * 3)(*box[0]), (C.c_double * 3)(*box[1]), C.byref(I)))
        self.cell_ptr = torch.empty(I.n_cells + 1, dtype=torch.int32, device=dev)
        self.occ = torch.empty(max(I.occ_bytes, 1), dtype=torch.uint8, device=dev)
        self.sorted = torch.empty(n, 4, dtype=torch.float32, device=dev)
        I.cell_ptr, I.occ, I.sorted = ptr(self.cell_ptr), ptr(self.occ), ptr(self.sorted)
        self.index = I
        nb = lib.xrd_nn_build_workspace_bytes(C.byref(I))
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check('xrd_nn_build', lib.xrd_nn_build(ptr(self.points), C.byref(I), ptr(ws), nb,
                                                   _stream(dev)))

    def query(self, queries, radius=None):
        """-> (dist f32 [Q], ids i32 [Q]) on the device; with a radius, targets further than it
        do not count (ids -1, dist inf)."""
        q = _pts(queries, self.device)
        dist = torch.empty(q.shape[0], dtype=torch.float32, device=self.device)
        ids = torch.empty(q.shape[0], dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            check('xrd_nn_query', _cabi.lib().xrd_nn_query(
                C.byref(self.index), ptr(q), q.shape[0], float(radius or 0.0), ptr(dist),
                ptr(ids), _stream(self.device)))
        return dist, ids


def _reduce_ws(n, dev):
    nb = _cabi.lib().xrd_eval_reduce_workspace_bytes(n)
    return torch.empty(nb, dtype=torch.uint8, device=dev), nb


def dist_stats(d, tau):
    """DEVICE f64 [3]: (sum d, sum d*d, count of d < tau), bit-identical run to run."""
    ws, nb = _reduce_ws(d.shape[0], d.device)
    out = torch.empty(3, dtype=torch.float64, device=d.device)
    with torch.cuda.device(d.device):
        check('xrd_eval_dist_stats', _cabi.lib().xrd_eval_dist_stats(
            ptr(d), d.shape[0], float(tau), ptr(out), ptr(ws), nb, _stream(d.device)))
    return out


def icp_stats(src, tgt, ids, dist):
    """DEVICE f64 [17]: (count, sum s, sum t, sum s t^T, sum d*d) over the correspondences."""
    ws, nb = _reduce_ws(src.shape[0], src.device)
    out = torch.empty(17, dtype=torch.float64, device=src.device)
    with torch.cuda.device(src.device):
        check('xrd_eval_icp_stats', _cabi.lib().xrd_eval_icp_stats(
            ptr(src), ptr(tgt), ptr(ids), ptr(dist), src.shape[0], ptr(out), ptr(ws), nb,
            _stream(src.device)))
    return out


def transform(points, T):
    """fp32(T applied in f64) to DEVICE points [n,3]; T a 4x4 (rows 0..2 used)."""
    T = np.ascontiguousarray(np.asarray(T, np.float64)[:3, :4]).reshape(-1)
    out = torch.empty_like(points)
    with torch.cuda.device(points.device):
        check('xrd_eval_transform', _cabi.lib().xrd_eval_transform(
            ptr(points), points.shape[0], (C.c_double * 12)(*T), ptr(out),
            _stream(points.device)))
    return out


# ---------------------------------------------------------------- ICP ---
def umeyama(stats):
    """Rigid Umeyama (no scaling) from the correspondence sums -> 4x4 f64; identity without
    correspondences."""
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


class RegistrationResult:
    def __init__(self, transformation, fitness, inlier_rmse, iterations):
        self.transformation = transformation
        self.fitness = fitness
        self.inlier_rmse = inlier_rmse
        self.iterations = iterations


def registration_icp(source, target, max_correspondence_distance=ICP_THRESHOLD, init=None,
                     max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, device=None):
    """open3d's point-to-point registration_icp (from memory, unverified): correspondences are
    each source point's nearest target within the distance; fitness = |C| / |S|, inlier_rmse =
    sqrt(sum d^2 / |C|); T <- Umeyama(C) T; stop after max_iteration updates or when fitness
    and rmse both change by less than the relative criteria.  The transform is applied to the
    original source once per iteration (f64, one fp32 rounding).  One host read per iteration
    (17 doubles).  -> RegistrationResult."""
    dev = _device(device) if not torch.is_tensor(source) or not source.is_cuda else source.device
    src = _pts(source, dev)
    index = target if isinstance(target, NNIndex) else NNIndex(target, dev)
    T = np.eye(4) if init is None else np.asarray(init, np.float64).copy()
    n = src.shape[0]

    def corr(T):
        s = transform(src, T)
        d, ids = index.query(s, max_correspondence_distance)
        st = icp_stats(s, index.points, ids, d).cpu().numpy()
        c = st[0]
        return st, (c / n if n else 0.0), (float(np.sqrt(st[16] / c)) if c else 0.0)

    st, fit, rmse = corr(T)
    it = 0
    for it in range(1, max_iteration + 1):
        T = umeyama(st) @ T
        st, f2, r2 = corr(T)
        done = abs(fit - f2) < relative_fitness and abs(rmse - r2) < relative_rmse
        fit, rmse = f2, r2
        if done:
            break
    return RegistrationResult(T, fit, rmse, it)


# ---------------------------------------------------------------- eval_recon.py ---
def _nn_dist(queries, targets):
    dev = _device(None) if not torch.is_tensor(targets) or not targets.is_cuda else targets.device
    return NNIndex(targets, dev).query(_pts(queries, dev))[0]


def completion_ratio(gt_points, rec_points, dist_th=0.05):
    """eval_recon.py:29-33: share of ground-truth points within dist_th of the reconstruction."""
    d = _nn_dist(gt_points, rec_points)
    return float(dist_stats(d, dist_th)[2].item() / d.shape[0])


def accuracy(gt_points, rec_points):
    """eval_recon.py:36-40: mean distance from the reconstruction to the ground truth."""
    d = _nn_dist(rec_points, gt_points)
    return float(dist_stats(d, 0.0)[0].item() / d.shape[0])


def completion(gt_points, rec_points):
    """eval_recon.py:43-47: mean distance from the ground truth to the reconstruction."""
    d = _nn_dist(gt_points, rec_points)
    return float(dist_stats(d, 0.0)[0].item() / d.shape[0])


def get_align_transformation(rec_meshfile, gt_meshfile, max_iteration=30, device=None):
    """ICP of the reconstruction's vertices onto the ground truth's (threshold 0.1, identity
    start).  eval_recon.py:50-63 uses 30 iterations, run_evaluation's copy 50."""
    dev = _device(device)
    rv, _ = load_mesh(rec_meshfile)
    gv, _ = load_mesh(gt_meshfile)
    return registration_icp(_pts(rv, dev), _pts(gv, dev), ICP_THRESHOLD,
                            max_iteration=max_iteration).transformation


def _aligned_vertices(rv, gv, transform_matrix, align, max_iteration_align):
    """The reconstruction's vertices after ds-eval's alignment: the given transform followed by
    a 30-iteration ICP, or (align) an ICP from the identity; the composite is applied once."""
    if transform_matrix is not None:
        T0 = np.asarray(transform_matrix, np.float64)
        icp = registration_icp(transform(rv, T0), gv, ICP_THRESHOLD, max_iteration=30)
        T = icp.transformation @ T0
    elif align:
        T = registration_icp(rv, gv, ICP_THRESHOLD,
                             max_iteration=max_iteration_align).transformation
    else:
        return rv, np.eye(4)
    return transform(rv, T), T


def calc_3d_metric(rec_meshfile, gt_meshfile, align=True, transform_matrix=None,
                   n_samples=N_SAMPLES, seed=0, uniforms=None, device=None):
    """eval_recon.py:93-136: align, sample n_samples points on each surface (trimesh
    sample_surface), -> accuracy / completion in cm and the 5 cm completion ratio in %.
    uniforms: optional (rec, gt) DEVICE f32 [n_samples,3] draws; else Philox seeds seed and
    seed + 1."""
    dev = _device(device)
    rv, rf = load_mesh(rec_meshfile)
    gv, gf = load_mesh(gt_meshfile)
    rv, gv = _pts(rv, dev), _pts(gv, dev)
    rv, _ = _aligned_vertices(rv, gv, transform_matrix, align, 30)
    ur, ug = (None, None) if uniforms is None else uniforms
    rec_pc, _ = sample_surface(rv, rf, n_samples, XRD_EVAL_TRIMESH, ur, seed, dev)
    gt_pc, _ = sample_surface(gv, gf, n_samples, XRD_EVAL_TRIMESH, ug, seed + 1, dev)
    d_rg = NNIndex(gt_pc, dev).query(rec_pc)[0]
    d_gr = NNIndex(rec_pc, dev).query(gt_pc)[0]
    a = dist_stats(d_rg, 0.05).cpu().numpy()
    c = dist_stats(d_gr, 0.05).cpu().numpy()
    return {'accuracy': a[0] / n_samples * 100, 'completion': c[0] / n_samples * 100,
            'completion ratio': c[2] / n_samples * 100}


def _cum_histogram(d, tau):
    """get_f1_score_histo's cumulative histogram on bins np.arange(0, 5 tau, tau / 100)."""
    edges = np.arange(0, tau * PLOT_STRETCH, tau / 100)
    e = torch.as_tensor(edges, dtype=torch.float64, device=d.device)
    x = d.double()
    b = torch.bucketize(x, e, right=True) - 1
    b = torch.where(x == e[-1], torch.full_like(b, len(edges) - 2), b)
    ok = (b >= 0) & (b < len(edges) - 1)
    hist = torch.bincount(b[ok], minlength=len(edges) - 1)
    return edges, (torch.cumsum(hist, 0).double() / d.shape[0]).cpu().numpy()


def fscore_from_distances(d1, d2, tau):
    """EvaluateHisto / get_f1_score_histo from DEVICE distances d1 (reconstruction -> ground
    truth) and d2 (ground truth -> reconstruction): precision, recall, F (0 when both are 0),
    the cumulative histograms and min / max / mean / median / std of both."""
    s1, s2 = dist_stats(d1, tau).cpu().numpy(), dist_stats(d2, tau).cpu().numpy()
    n1, n2 = d1.shape[0], d2.shape[0]
    p, r = s1[2] / n1, s2[2] / n2
    f = 2 * r * p / (r + p) if r + p > 0 else 0.0
    out = dict(precision=p, recall=r, fscore=f, mean1=s1[0] / n1, mean2=s2[0] / n2)
    for k, d in (('1', d1), ('2', d2)):
        x = d.double()
        out['min' + k] = float(x.min())
        out['max' + k] = float(x.max())
        out['median' + k] = float(x.sort().values[(x.numel() - 1) // 2: x.numel() // 2 + 1].mean())
        out['std' + k] = float(x.std(unbiased=False))
    out['edges_source'], out['cum_source'] = _cum_histogram(d1, tau)
    out['edges_target'], out['cum_target'] = _cum_histogram(d2, tau)
    return out


def fscore_distances(rec_v, rec_f, gt_v, gt_f, seed=0, uniforms=None, device=None):
    """run_evaluation:180-201 and EvaluateHisto's distances: the mesh with fewer vertices is
    sampled (open3d sample_points_uniformly) with as many points as the other has vertices;
    d1 is then the reconstruction's vertices to the ground truth's point set and d2 the ground
    truth's point set to the reconstruction's vertices when the ground truth has fewer vertices,
    otherwise d1 = reconstruction vertices -> ground-truth vertices and d2 = ground-truth
    vertices -> reconstruction samples (EvaluateHisto replaces the sampled side's distances by
    its vertices' for the colour meshes before computing the F-score).  -> (d1, d2, branch)."""
    dev = _device(device)
    rv, gv = _pts(rec_v, dev), _pts(gt_v, dev)
    if gv.shape[0] < rv.shape[0]:
        gt_pcd, _ = sample_surface(gv, gt_f, rv.shape[0], XRD_EVAL_OPEN3D, uniforms, seed, dev)
        d1 = NNIndex(gt_pcd, dev).query(rv)[0]
        d2 = NNIndex(rv, dev).query(gv)[0]
        return d1, d2, 'sample_gt'
    pcd, _ = sample_surface(rv, rec_f, gv.shape[0], XRD_EVAL_OPEN3D, uniforms, seed, dev)
    d1 = NNIndex(gv, dev).query(rv)[0]
    d2 = NNIndex(pcd, dev).query(gv)[0]
    return d1, d2, 'sample_rec'


def run_evaluation(pred_ply, path_to_pred_ply, scene, distance_thresh=0.01,
                   transform_matrix=None, icp_align=True, full_path_to_gt_ply=None, seed=0,
                   uniforms=None, device=None):
    """evaluate_3d_reconstruction.py:75-276 without the plots: align (the given transform then a
    30-iteration ICP, or a 50-iteration ICP), write trans_mesh.ply next to the prediction, and
    the precision / recall / F-score files under <path>/<pred_ply without .ply>/."""
    dev = _device(device)
    if full_path_to_gt_ply is None:
        raise ValueError('full_path_to_gt_ply is required (no ground-truth database here)')
    pred_path = os.path.join(path_to_pred_ply, pred_ply)
    out_dir = os.path.join(path_to_pred_ply, pred_ply[:-4])
    os.makedirs(out_dir, exist_ok=True)
    rv, rf = load_mesh(pred_path)
    gv, gf = load_mesh(full_path_to_gt_ply)
    rv, gv = _pts(rv, dev), _pts(gv, dev)
    if transform_matrix is not None or icp_align:
        rv, _ = _aligned_vertices(rv, gv, transform_matrix, icp_align, 50)
        from .io_formats import write_ply
        write_ply(os.path.join(path_to_pred_ply, 'trans_mesh.ply'), rv.cpu().numpy(), rf)
    d1, d2, _ = fscore_distances(rv, rf, gv, gf, seed, uniforms, dev)
    h = fscore_from_distances(d1, d2, distance_thresh)
    base = os.path.join(out_dir, scene)
    np.savetxt(base + '.recall.txt', h['cum_target'])
    np.savetxt(base + '.precision.txt', h['cum_source'])
    np.savetxt(base + '.prf_tau_plotstr.txt',
               np.array([h['precision'], h['recall'], h['fscore'], distance_thresh,
                         PLOT_STRETCH]))
    np.savetxt(base + '.min12_max12_mean12_median12_std12.txt',
               np.array([h['min1'], h['min2'], h['max1'], h['max2'], h['mean1'], h['mean2'],
                         h['median1'], h['median2'], h['std1'], h['std2']]))
    return {'dist_threshold': distance_thresh, 'precision': h['precision'],
            'recall': h['recall'], 'f-score': h['fscore'], 'mean precision': h['mean1'],
            'mean recall': h['mean2']}


def calc_3d_metric_New(rec_meshfile, gt_meshfile, align=True, distance_thresh=0.01,
                       transform_matrix=None, seed=0, uniforms=None, device=None):
    """eval_recon.py:139-155: run_evaluation on the mesh file, scene = the ground truth's name."""
    rec_meshfile = str(rec_meshfile)
    gt_meshfile = str(gt_meshfile)
    return run_evaluation(os.path.basename(rec_meshfile), os.path.dirname(rec_meshfile),
                          os.path.basename(gt_meshfile)[:-4], distance_thresh=distance_thresh,
                          transform_matrix=transform_matrix, icp_align=align,
                          full_path_to_gt_ply=gt_meshfile, seed=seed, uniforms=uniforms,
                          device=device)


# ---------------------------------------------------------------- calc_2d_metric ---
RENDER_W = RENDER_H = 500   # calc_2d_metric's camera: 500 x 500, focal 300, centre 249.5
RENDER_FOCAL = 300.0
Z_FAR = 20.0                # set_constant_z_far(20)
NEAR_FRACTION = 0.01        # open3d's z_near: 0.01 x the drawn geometry's largest AABB extent


def _norm(x):
    x = np.asarray(x, np.float64)
    return np.sqrt((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2])


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def normalize(x):
    """eval_recon.py:16-17, over the last axis of [..., 3] with an explicit sum order, so one
    vector and a batch of them round alike."""
    x = np.asarray(x, np.float64)
    return x / _norm(x)[..., None]


def viewmatrix(z, up, pos):
    """eval_recon.py:20-26: [..., 3, 4] camera-to-world columns (x, y, z, position) with z along
    `z`, built from `up`."""
    vec2 = normalize(z)
    up = np.broadcast_to(np.asarray(up, np.float64), vec2.shape)
    vec0 = normalize(_cross(up, vec2))
    vec1 = normalize(_cross(vec2, vec0))
    pos = np.broadcast_to(np.asarray(pos, np.float64), vec2.shape)
    return np.stack([vec0, vec1, vec2, pos], -1)


def volume_rectangular(extents, count, transform=None, rng=None):
    """trimesh.sample.volume_rectangular (from memory, unverified): (random((count, 3)) - 0.5) *
    extents, then transform (4x4) applied as ((T0 x + T1 y) + T2 z) + T3 per row.  `rng` is a
    numpy RandomState (the global one when None); count rows are the same draws as count
    one-row calls."""
    rng = np.random if rng is None else rng
    p = (rng.random((count, 3)) - 0.5) * np.asarray(extents, np.float64)
    if transform is None:
        return p
    T = np.asarray(transform, np.float64)
    return np.stack([((T[a, 0] * p[:, 0] + T[a, 1] * p[:, 1]) + T[a, 2] * p[:, 2]) + T[a, 3]
                     for a in range(3)], -1)


def _min_area_rect(p2):
    """Smallest-area rectangle around 2D points over their hull's edge directions ->
    (area, unit edge direction)."""
    from scipy.spatial import ConvexHull
    h = p2[ConvexHull(p2).vertices]
    e = np.roll(h, -1, 0) - h
    e = e / np.linalg.norm(e, axis=1, keepdims=True)
    best = (np.inf, None)
    for d in e:
        r = h @ np.array([d, [-d[1], d[0]]]).T
        area = np.ptp(r[:, 0]) * np.ptp(r[:, 1])
        if area < best[0]:
            best = (area, d)
    return best


def oriented_bounds(obj, angle_digits=1, ordered=True):
    """trimesh.bounds.oriented_bounds, restated from memory (unverified): the minimum-volume box
    over the convex hull's face normals, each with the minimum-area rectangle of the points
    projected on the normal's plane.  obj: a mesh, vertices or a PLY path.  -> (to_origin 4x4
    mapping the box's centre to the origin and its axes to x, y, z; extents), extents ascending
    when `ordered`.  angle_digits is accepted for the reference's signature; normals are merged
    to 1e-8."""
    from scipy.spatial import ConvexHull
    v, _ = load_mesh(obj) if not isinstance(obj, np.ndarray) else (obj, None)
    pts = np.asarray(v.cpu().numpy() if torch.is_tensor(v) else v, np.float64).reshape(-1, 3)
    hull = ConvexHull(pts)
    hv = pts[hull.vertices]
    normals = np.unique(np.round(hull.equations[:, :3], 8), axis=0)
    best = (np.inf, None)
    for n in normals:
        n = n / np.linalg.norm(n)
        a = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        a /= np.linalg.norm(a)
        b = np.cross(n, a)
        area, d = _min_area_rect(hv @ np.stack([a, b]).T)
        vol = area * np.ptp(hv @ n)
        if vol < best[0]:
            u = d[0] * a + d[1] * b
            best = (vol, np.stack([n, u, np.cross(n, u)]))
    R = best[1]
    proj = hv @ R.T
    lo, hi = proj.min(0), proj.max(0)
    extents = hi - lo
    centre = R.T @ ((lo + hi) / 2)
    if ordered:
        order = np.argsort(extents, kind='stable')
        R, extents = R[order], extents[order]
    if np.linalg.det(R) < 0:
        R[2] *= -1
    to_origin = np.eye(4)
    to_origin[:3, :3] = R
    to_origin[:3, 3] = -R @ centre
    return to_origin, extents


def get_cam_position(gt_meshfile):
    """eval_recon.py:158-166: the box camera origins are drawn from, inside the ground truth's
    oriented bounds (extents scaled by 0.3, 0.7, 0.7, centre raised 0.4 m in world z)."""
    to_origin, extents = oriented_bounds(gt_meshfile)
    extents = extents.copy()
    extents[2] *= 0.7
    extents[1] *= 0.7
    extents[0] *= 0.3
    transform = np.linalg.inv(to_origin)
    transform[2, 3] += 0.4
    return extents, transform


def _camera(near, H=RENDER_H, W=RENDER_W, fx=RENDER_FOCAL, fy=RENDER_FOCAL, cx=None, cy=None,
            far=Z_FAR):
    cx = H / 2.0 - 0.5 if cx is None else cx
    cy = W / 2.0 - 0.5 if cy is None else cy
    return _cabi.XrdEvalCamera(H, W, fx, fy, cx, cy, near, far)


def points_seen(points, c2w, W=RENDER_W, H=RENDER_H, fx=RENDER_FOCAL, fy=RENDER_FOCAL, cx=None,
                cy=None, device=None):
    """check_proj for K views at once: DEVICE or host points [N,3], c2w [K,4,4] -> bool [K]
    (host), True where some point projects into the view (xrd_eval_points_seen)."""
    dev = _device(device) if not torch.is_tensor(points) or not points.is_cuda else points.device
    p = _pts(points, dev)
    c = np.array(c2w, np.float64, copy=True).reshape(-1, 4, 4)
    c[:, :3, 1] *= -1.0
    c[:, :3, 2] *= -1.0
    w2c = torch.from_numpy(np.ascontiguousarray(np.linalg.inv(c).astype(np.float32)[:, :3, :4]))
    w2c = w2c.to(dev)
    seen = torch.empty(len(c), dtype=torch.uint8, device=dev)
    cam = _camera(0.0, H, W, fx, fy, cx, cy, 1.0)
    with torch.cuda.device(dev):
        check('xrd_eval_points_seen', _cabi.lib().xrd_eval_points_seen(
            ptr(p), p.shape[0], ptr(w2c), len(c), C.byref(cam), ptr(seen), _stream(dev)))
    return seen.cpu().numpy().astype(bool)


def check_proj(points, W, H, fx, fy, cx, cy, c2w):
    """eval_recon.py:66-90: whether any point projects into the view c2w [4,4]."""
    return bool(points_seen(points, np.asarray(c2w)[None], W, H, fx, fy, cx, cy)[0])


def sample_views(pc_unseen, extents, transform, n_imgs, seed=0, batch=1024, max_candidates=None,
                 device=None, seen_fn=None):
    """calc_2d_metric's view sampler (eval_recon.py:212-232): origin in the camera box (numpy
    RandomState(seed)), target = three round(uniform(-1e4, 1e4), 2) (random.Random(seed)) minus
    the origin, up (0, 0, -1); a view that sees the unseen cloud is drawn again.  Candidates are
    drawn and checked `batch` at a time and taken in order; the two streams are independent, so
    the accepted views are those of the one-at-a-time loop.  -> c2w f64 [n_imgs,4,4].  Raises
    RuntimeError after max_candidates (default 1000 n_imgs) candidates.  seen_fn(c2w [K,4,4]) ->
    bool [K] replaces the device check (xrd_eval_points_seen on pc_unseen) when given."""
    import random
    pyr, npr = random.Random(seed), np.random.RandomState(seed)
    if seen_fn is None:
        dev = _device(device)
        pts = _pts(pc_unseen, dev)
        seen_fn = (lambda c: points_seen(pts, c, device=dev)) if pts.shape[0] else \
            (lambda c: np.zeros(len(c), bool))
    limit = 1000 * n_imgs if max_candidates is None else max_candidates
    views, tried = [], 0
    while len(views) < n_imgs:
        k = min(batch, limit - tried)
        if k <= 0:
            raise RuntimeError(f'calc_2d_metric: {tried} candidate views all see the unseen '
                               f'region; {len(views)} of {n_imgs} accepted')
        origin = volume_rectangular(extents, k, transform, npr)
        target = np.array([[round(pyr.uniform(-10000, +10000), 2) for _ in range(3)]
                           for _ in range(k)]) - origin
        c2w = np.tile(np.eye(4), (k, 1, 1))
        c2w[:, :3, :] = viewmatrix(target, [0, 0, -1], origin)
        seen = np.asarray(seen_fn(c2w), bool)
        tried += k
        for i in np.nonzero(~seen)[0][:n_imgs - len(views)]:
            views.append(c2w[i])
    return np.array(views).reshape(-1, 4, 4)


class DepthRenderer:
    """xrd_eval_render_depth over one mesh: DEVICE vertices / faces, near = 0.01 x the largest
    AABB extent of the vertices (one host read), far 20; renders up to 32 views per launch."""

    def __init__(self, verts, faces, device=None, H=RENDER_H, W=RENDER_W, fx=RENDER_FOCAL,
                 fy=RENDER_FOCAL, cx=None, cy=None, near=None, far=Z_FAR):
        dev = _device(device) if not torch.is_tensor(verts) or not verts.is_cuda else verts.device
        self.device = dev
        self.verts = _pts(verts, dev)
        f = faces if torch.is_tensor(faces) else torch.from_numpy(np.asarray(faces, np.int32))
        self.faces = f.to(dev, torch.int32).reshape(-1, 3).contiguous()
        if near is None:
            lo, hi = torch.aminmax(self.verts, dim=0)
            near = NEAR_FRACTION * float((hi - lo).max())
        self.camera = _camera(near, H, W, fx, fy, cx, cy, far)
        self.B = _cabi.XRD_EVAL_RENDER_MAX_VIEWS
        self.ws_bytes = _cabi.lib().xrd_eval_render_workspace_bytes(self.faces.shape[0], self.B)
        if self.ws_bytes == 0:
            raise ValueError('the depth renderer needs at least one face')
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=dev)

    def render(self, w2c, out=None, status=None):
        """w2c [n,3,4] or [n,4,4] (host f64 or DEVICE) -> DEVICE depth f32 [n,H,W].  status: a
        DEVICE i32 [>= ceil(n / 32)] to collect the per-launch status words in (the caller
        checks them); without it they are read at once."""
        W = torch.as_tensor(np.asarray(w2c, np.float64) if not torch.is_tensor(w2c) else w2c)
        W = W.to(self.device, torch.float64)[:, :3, :4].contiguous()
        n = W.shape[0]
        cam = self.camera
        out = torch.empty(n, cam.H, cam.W, dtype=torch.float32, device=self.device) \
            if out is None else out
        own = status is None
        if own:
            status = torch.zeros(max(1, -(-n // self.B)), dtype=torch.int32, device=self.device)
        lib = _cabi.lib()
        with torch.cuda.device(self.device):
            s = _stream(self.device)
            for k, b0 in enumerate(range(0, n, self.B)):
                nb = min(self.B, n - b0)
                check('xrd_eval_render_depth', lib.xrd_eval_render_depth(
                    ptr(self.verts), self.verts.shape[0], ptr(self.faces), self.faces.shape[0],
                    ptr(W[b0:b0 + nb]), nb, C.byref(cam), ptr(out[b0:b0 + nb]),
                    ptr(status[k:k + 1]), ptr(self.ws), self.ws_bytes, s))
        if own:
            _check_status(status)
        return out


def _check_status(status):
    st = status.cpu().numpy()
    if st.any():
        check('xrd_eval_render_depth', int(st[st != 0][0]))


def depth_l1_sums(gt, rec):
    """DEVICE f64 [n,2] = (sum |gt - rec|, count) over rec > 0 per view, bit-identical run to
    run (xrd_eval_depth_l1)."""
    n = gt.shape[0]
    out = torch.empty(n, 2, dtype=torch.float64, device=gt.device)
    with torch.cuda.device(gt.device):
        check('xrd_eval_depth_l1', _cabi.lib().xrd_eval_depth_l1(
            ptr(gt), ptr(rec), n, gt[0].numel() if n else 0, ptr(out), _stream(gt.device)))
    return out


def unseen_file(gt_meshfile):
    """The unseen point cloud calc_2d_metric reads beside the ground-truth mesh."""
    return str(gt_meshfile).replace('.ply', '_pc_unseen.npy')


def calc_2d_metric(rec_meshfile, gt_meshfile, transform_matrix=None, align=True, n_imgs=1000,
                   seed=0, device=None):
    """eval_recon.py:169-283, depth L1 in cm: align the reconstruction as calc_3d_metric does,
    draw n_imgs views inside the ground truth's camera box that do not see
    <gt>_pc_unseen.npy, render both meshes' depth at 500 x 500 (fx = fy = 300) and average, over
    the views where the reconstruction draws anything, the mean |gt - rec| over its pixels.
    -> {'depth l1': cm} (NaN when no view draws the reconstruction).  Renders run 32 views per
    launch; the host reads the sums once.  The reference reads a quantised OpenGL depth buffer
    and keeps whichever surface wins z-fighting; here z is exact and the nearest surface wins."""
    dev = _device(device)
    pc_unseen = np.load(unseen_file(gt_meshfile))
    rv, rf = load_mesh(rec_meshfile)
    gv, gf = load_mesh(gt_meshfile)
    rv, gv = _pts(rv, dev), _pts(gv, dev)
    rv, _ = _aligned_vertices(rv, gv, transform_matrix, align, 30)
    extents, transform = get_cam_position(gv.cpu().numpy())
    c2w = sample_views(pc_unseen, extents, transform, n_imgs, seed, device=dev)
    if n_imgs == 0:
        return {'depth l1': float('nan')}
    w2c = np.linalg.inv(c2w)
    gt_r, rec_r = DepthRenderer(gv, gf, dev), DepthRenderer(rv, rf, dev)
    B = gt_r.B
    nbatch = -(-n_imgs // B)
    sums = torch.empty(n_imgs, 2, dtype=torch.float64, device=dev)
    status = torch.zeros(2 * nbatch, dtype=torch.int32, device=dev)
    for k in range(nbatch):
        sl = slice(k * B, min(n_imgs, (k + 1) * B))
        gd = gt_r.render(w2c[sl], status=status[2 * k:2 * k + 1])
        rd = rec_r.render(w2c[sl], status=status[2 * k + 1:2 * k + 2])
        sums[sl] = depth_l1_sums(gd, rd)
    _check_status(status)
    s = sums.cpu().numpy()
    ok = s[:, 1] > 0
    if not ok.any():
        return {'depth l1': float('nan')}
    return {'depth l1': float((s[ok, 0] / s[ok, 1]).mean() * 100)}
