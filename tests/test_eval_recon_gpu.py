"""ds-eval reconstruction metrics on the device (csrc/eval.cu, xrdslam_b200/eval_recon.py):
samplers, nearest-neighbour queries, reductions, transform and ICP bit for bit against the numpy
restatement (oracle/eval_recon.py), distances against scipy's cKDTree, status codes, and
EvalMatrics end to end on the synthetic room."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import eval_recon as oe

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
pytestmark = pytest.mark.gpu
f32 = np.float32


def _bits(t):
    return (t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t)).view(np.uint32)


def _room(spacing=0.1):
    from xrdslam_b200.synthetic import room_mesh
    return room_mesh(spacing)


# ---- sampling --------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [0, 1])
def test_samplers_bit_exact_with_given_uniforms(cuda_dev, mode):
    from xrdslam_b200.eval_recon import sample_surface
    v, f = _room(0.1)
    n = 30011
    U = np.random.default_rng(mode).random((n, 3 if mode == 0 else 2), dtype=f32)
    p, fi = sample_surface(v, f, n, mode, torch.from_numpy(U).to(cuda_dev), device=cuda_dev)
    po, fo = oe.sample_trimesh(v, f, U) if mode == 0 else oe.sample_open3d(v, f, n, U)
    assert np.array_equal(fi.cpu().numpy(), fo)
    assert np.array_equal(_bits(p), po.astype(f32).view(np.uint32))


@pytest.mark.parametrize('mode', [0, 1])
def test_philox_samples_lie_on_their_faces_with_area_weighted_counts(cuda_dev, mode):
    from scipy.stats import chisquare
    from xrdslam_b200.eval_recon import sample_surface
    v, f = _room(0.5)
    n = 400000
    p, fi = sample_surface(v, f, n, mode, None, seed=11, device=cuda_dev)
    p, fi = p.cpu().numpy().astype(np.float64), fi.cpu().numpy()
    U = oe.philox_uniforms(11, n, 3 if mode == 0 else 2)
    po, fo = oe.sample_trimesh(v, f, U) if mode == 0 else oe.sample_open3d(v, f, n, U)
    assert np.array_equal(fi, fo) and np.array_equal(p.astype(f32), po)   # Philox restated
    V = v.astype(np.float64)
    a, b, c = V[f[fi, 0]], V[f[fi, 1]], V[f[fi, 2]]
    nrm = np.cross(b - a, c - a)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    assert np.abs(((p - a) * nrm).sum(1)).max() <= 1e-6
    # barycentric coordinates in [0, 1]
    e1, e2, e = b - a, c - a, p - a
    d11, d12, d22 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
    d1, d2 = (e * e1).sum(1), (e * e2).sum(1)
    den = d11 * d22 - d12 * d12
    w1, w2 = (d22 * d1 - d12 * d2) / den, (d11 * d2 - d12 * d1) / den
    tol = 1e-5
    assert w1.min() >= -tol and w2.min() >= -tol and (w1 + w2).max() <= 1 + tol
    cum, tot = oe.area_prefix(v, f)
    area = np.diff(np.concatenate([[0.0], cum]))
    counts = np.bincount(fi, minlength=len(f))
    exp = area / tot * n
    assert chisquare(counts, exp).pvalue > 1e-3


@pytest.mark.parametrize('case', ['no_faces', 'zero_area', 'bad_index', 'negative_index',
                                  'nan_vertex', 'inf_vertex'])
def test_invalid_meshes_raise(cuda_dev, case):
    from xrdslam_b200._cabi import XrdError
    from xrdslam_b200.eval_recon import sample_surface
    v, f = _room(1.0)
    v, f = v.copy(), f.copy()
    if case == 'no_faces':
        f = f[:0]
    elif case == 'zero_area':
        f[:] = f[:, :1]
    elif case == 'bad_index':
        f[3, 1] = len(v)
    elif case == 'negative_index':
        f[0, 2] = -1
    elif case == 'nan_vertex':
        v[5, 0] = np.nan
    else:
        v[7, 2] = np.inf
    with pytest.raises(XrdError, match='XRD_E_SHAPE'):
        sample_surface(v, f, 100, 0, None, device=cuda_dev)


def test_workspace_too_small_and_null(cuda_dev):
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    d = torch.rand(10000, device=cuda_dev)
    out = torch.empty(3, dtype=torch.float64, device=cuda_dev)
    nb = lib.xrd_eval_reduce_workspace_bytes(10000)
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda_dev)
    s = torch.cuda.current_stream().cuda_stream
    assert lib.xrd_eval_dist_stats(d.data_ptr(), 10000, 0.5, out.data_ptr(), ws.data_ptr(),
                                   nb - 1, s) == -3
    assert lib.xrd_eval_dist_stats(None, 10000, 0.5, out.data_ptr(), ws.data_ptr(), nb, s) == -6
    v, f = _room(1.0)
    nbs = lib.xrd_eval_surface_workspace_bytes(len(f))
    with pytest.raises(_cabi.XrdError, match='XRD_E_WORKSPACE'):
        _cabi.check('xrd_eval_surface_prepare', lib.xrd_eval_surface_prepare(
            1, len(v), 1, len(f), 1, 1, 1, 1, nbs - 1, s))


# ---- nearest neighbour -----------------------------------------------------------------------
def _nn_cases():
    rng = np.random.default_rng(5)
    v, f = _room(0.1)
    surf = oe.sample_trimesh(v, f, rng.random((20000, 3), dtype=f32))[0]
    q = oe.sample_trimesh(v, f, rng.random((20000, 3), dtype=f32))[0]
    q = q + rng.normal(0, 0.01, q.shape).astype(f32)
    far = q.copy()
    k = len(q) // 10
    dirs = rng.normal(size=(k, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    far[:k] = (far[:k] + dirs * rng.uniform(0.5, 3.0, (k, 1))).astype(f32)
    dup = surf.copy()
    dup[15000:] = dup[:5000]
    outside = rng.uniform(-8, 8, (20000, 3)).astype(f32)
    return {
        'surface': (surf, q),
        'far_outliers': (surf, far),
        'duplicates': (dup, np.concatenate([dup[:3000], q[:17000]])),
        'outside_box': (surf, outside),
        'offset_10m': (surf + f32(10), q + f32(10)),
        'single_target': (surf[:1], q[:5000]),
        'one_query': (surf, q[:1]),
        'planar_lattice': (np.stack(np.meshgrid(np.arange(150) * 0.01, np.arange(150) * 0.01,
                                                [0.0], indexing='ij'), -1).reshape(-1, 3)
                           .astype(f32), q[:5000] * f32(0.3)),
    }


@pytest.mark.parametrize('case', list(_nn_cases().keys()))
def test_unbounded_nn_bit_exact_against_brute_force(cuda_dev, case):
    from xrdslam_b200 import _cabi
    from xrdslam_b200.eval_recon import NNIndex
    P, Q = _nn_cases()[case]
    idx = NNIndex(torch.from_numpy(P).to(cuda_dev))
    cnt = torch.zeros(2, dtype=torch.int64, device=cuda_dev)
    _cabi.lib().xrd_debug_nn_counters(cnt.data_ptr())
    try:
        d, i = idx.query(torch.from_numpy(Q).to(cuda_dev))
    finally:
        _cabi.lib().xrd_debug_nn_counters(None)
    do, io = oe.nn_brute(Q, P)
    assert np.array_equal(i.cpu().numpy(), io)
    assert np.array_equal(_bits(d), do.view(np.uint32))
    # the result does not depend on how the queries are split over launches
    h = len(Q) // 3
    parts = [idx.query(torch.from_numpy(Q[s:e]).to(cuda_dev)) for s, e in ((0, h), (h, len(Q)))]
    assert np.array_equal(torch.cat([p[1] for p in parts]).cpu().numpy(), io)
    nodes, pts = cnt.tolist()
    print(f'{case}: {len(P)} x {len(Q)}: {nodes / len(Q):.1f} nodes, {pts / len(Q):.1f} points '
          'per query')
    assert pts < len(P) * len(Q) / 20 or len(P) < 100


def test_radius_nn_bit_exact_including_the_radius(cuda_dev):
    from xrdslam_b200.eval_recon import NNIndex
    P, Q = _nn_cases()['far_outliers']
    Q = np.concatenate([Q, P[:100] + np.array([0.1, 0, 0], f32), P[100:200] - np.array(
        [0, 0, 0.1], f32)])
    idx = NNIndex(torch.from_numpy(P).to(cuda_dev))
    for r in (0.1, 0.02):
        d, i = idx.query(torch.from_numpy(Q).to(cuda_dev), r)
        do, io = oe.nn_brute(Q, P, radius=r)
        assert np.array_equal(i.cpu().numpy(), io)
        assert np.array_equal(_bits(d), do.view(np.uint32))
        assert (io == -1).any() and (io >= 0).any()
    # a target exactly at the radius counts
    idx1 = NNIndex(torch.tensor([[0.1, 0.0, 0.0]], device=cuda_dev))
    d, i = idx1.query(torch.zeros(1, 3, device=cuda_dev), 0.1)
    assert i.item() == 0


def test_nn_against_ckdtree_at_200k(cuda_dev):
    from xrdslam_b200.eval_recon import NNIndex
    rng = np.random.default_rng(9)
    v, f = _room(0.1)
    P = oe.sample_trimesh(v, f, rng.random((200000, 3), dtype=f32))[0]
    Q = oe.sample_trimesh(v, f, rng.random((200000, 3), dtype=f32))[0] + rng.normal(
        0, 0.02, (200000, 3)).astype(f32)
    d, _ = NNIndex(torch.from_numpy(P).to(cuda_dev)).query(torch.from_numpy(Q).to(cuda_dev))
    d64, _ = oe.ckdtree_dist(Q, P)
    assert np.abs(d.cpu().numpy().astype(np.float64) - d64).max() <= 1e-5


# ---- reductions, transform, ICP --------------------------------------------------------------
def test_reductions_bit_identical_and_match_restatement(cuda_dev):
    from xrdslam_b200.eval_recon import NNIndex, dist_stats, icp_stats
    P, Q = _nn_cases()['far_outliers']
    idx = NNIndex(torch.from_numpy(P).to(cuda_dev))
    q = torch.from_numpy(Q).to(cuda_dev)
    d, i = idx.query(q, 0.1)
    d_unb, _ = idx.query(q)
    a = [dist_stats(d_unb, 0.01).cpu().numpy() for _ in range(2)]
    assert np.array_equal(a[0], a[1])
    assert np.array_equal(a[0], oe.dist_stats(d_unb.cpu().numpy(), 0.01))
    b = [icp_stats(q, idx.points, i, d).cpu().numpy() for _ in range(2)]
    assert np.array_equal(b[0], b[1])
    assert np.array_equal(b[0], oe.icp_stats(Q, P, i.cpu().numpy(), d.cpu().numpy()))
    # queries split over two launches give the same distances, hence the same sums
    h = 7777
    d2 = torch.cat([idx.query(q[:h])[0], idx.query(q[h:])[0]])
    assert np.array_equal(dist_stats(d2, 0.01).cpu().numpy(), a[0])


def test_transform_bit_exact(cuda_dev):
    from xrdslam_b200.eval_recon import transform
    v, _ = _room(0.1)
    T = np.eye(4)
    T[:3, :3] = np.linalg.qr(np.random.default_rng(2).normal(size=(3, 3)))[0]
    T[:3, 3] = [10.1, -3.3, 0.7]
    out = transform(torch.from_numpy(v).to(cuda_dev), T)
    assert np.array_equal(_bits(out), oe.transform(v, T).view(np.uint32))


def test_device_icp_matches_oracle_icp(cuda_dev):
    from test_eval_recon_cpu import _rot
    from xrdslam_b200.eval_recon import registration_icp
    v, _ = _room(0.25)
    T = np.eye(4)
    T[:3, :3] = _rot(2.0, [0.3, -0.5, 1.0])
    T[:3, 3] = [0.03, -0.01, 0.02]
    src = oe.transform(v, np.linalg.inv(T))
    for it in (50, 3):
        r = registration_icp(torch.from_numpy(src).to(cuda_dev), torch.from_numpy(v).to(cuda_dev),
                             0.1, max_iteration=it)
        ro = oe.registration_icp(src, v, 0.1, max_iteration=it, nn=oe.nn_kdtree_f32)
        assert r.iterations == ro['iterations']
        assert abs(r.fitness - ro['fitness']) <= 1e-4
        assert np.abs(r.transformation - ro['transformation']).max() <= 1e-5
        if it == 50:
            assert r.iterations < 50 and np.abs(r.transformation - T).max() < 1e-4
    assert ro['iterations'] == 3


# ---- end to end ------------------------------------------------------------------------------
class _KF:
    def __init__(self, c2w, rgb, depth):
        self._pose = torch.as_tensor(c2w)
        self.rgb, self.depth = rgb, depth

    def get_pose(self):
        return self._pose


class _Algo:
    def __init__(self, gt, est):
        self.gt, self.est = gt, est

    def get_gt_c2w_list_ori(self):
        return self.gt

    def get_gt_c2w_list(self):
        return self.gt

    def get_estimate_c2w_list(self):
        return self.est


def test_eval_matrics_end_to_end(cuda_dev, tmp_path):
    import make_golden_cull as mg
    from xrdslam_b200 import io_formats
    from xrdslam_b200.common import cull_mesh, get_mesh_from_RGBD
    from xrdslam_b200.eval import EvalMatrics
    from xrdslam_b200.mesher import TriMesh
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(8, width=160, height=120)
    kfs = [_KF(p, rgb, d) for p, (rgb, d) in zip(poses, frames)]
    mesh = get_mesh_from_RGBD(cam, kfs, device=cuda_dev)
    host = TriMesh(mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy())
    depth = np.stack([d for _, d in frames]).astype(f32)
    ds = mg.Dataset(depth, np.stack(poses).astype(f32),
                    [cam.height, cam.width, cam.fx, cam.fy, cam.cx, cam.cy])
    culled = cull_mesh(ds, host, None, eval_rec=True, device=cuda_dev)
    culled.export(str(tmp_path / 'final_mesh_rec.ply'))
    gt = [torch.as_tensor(p) for p in poses]
    est = [g.clone() for g in gt]
    for e in est:
        e[:3, 3] += torch.tensor([0.002, -0.001, 0.0])
    io_formats.save_eval_tar(_Algo(gt, est), str(tmp_path), len(gt))
    gv, gf = _room(0.05)
    gt_path = io_formats.write_ply(str(tmp_path / 'room_gt.ply'), gv, gf)
    m = EvalMatrics(output_dir=tmp_path, gt_mesh=gt_path, seed=4)
    res = m.main()
    _, T = m.trajectory()
    rv, rf, _ = io_formats.read_ply(str(tmp_path / 'final_mesh_rec.ply'))
    exp = oe.ds_eval_3d(rv, rf, gv, gf, T, seed=4, tau=0.01)
    for k, e in exp.items():
        assert abs(res[k] - e) <= 1e-6 * max(abs(e), 1e-12), (k, res[k], e)
    print({k: round(float(v), 5) for k, v in res.items()})
    # rec samples -> 200k ground-truth samples: bounded by the samples' spacing (~1.5 cm on the
    # room's 193 m^2), so the TSDF surface error shows in the vertex distances below
    assert res['accuracy'] / 100 < 0.03
    assert res['mean precision'] < 0.05
    assert res['completion ratio'] < 100
    out = tmp_path / 'final_mesh_rec'
    assert os.path.exists(tmp_path / 'trans_mesh.ply')
    for name in ('recall', 'precision'):
        cum = np.loadtxt(out / f'room_gt.{name}.txt')
        assert cum.ndim == 1 and len(cum) >= 499 and np.all(np.diff(cum) >= 0)
    prf = np.loadtxt(out / 'room_gt.prf_tau_plotstr.txt')
    assert np.allclose(prf[:3], [res['precision'], res['recall'], res['f-score']])
    assert np.loadtxt(out / 'room_gt.min12_max12_mean12_median12_std12.txt').shape == (10,)
