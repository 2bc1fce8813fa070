"""ds-eval depth L1 on the device (csrc/eval_render.cu, eval_recon.calc_2d_metric): depth maps
bit for bit against the numpy rasteriser (oracle/eval_render.py), watertightness at 1 cm
spacing, the unseen check and the per-view sums against their restatements, status codes, and
calc_2d_metric / EvalMatrics end to end on the synthetic room."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import eval_render as ore

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
pytestmark = pytest.mark.gpu
f32 = np.float32
NO_UNSEEN = np.zeros((0, 3), f32)


def _cam(H, W, fx, fy, cx, cy, near=0.063, far=20.0):
    return dict(H=H, W=W, fx=fx, fy=fy, cx=cx, cy=cy, near=near, far=far)


def _views(verts, n, seed, pc=NO_UNSEEN):
    from xrdslam_b200.eval_recon import get_cam_position, sample_views
    ext, T = get_cam_position(verts)
    return sample_views(pc, ext, T, n, seed=seed, seen_fn=lambda c: np.array(
        [ore.check_proj(pc, 500, 500, 300., 300., 249.5, 249.5, x) for x in c]) if len(pc)
        else np.zeros(len(c), bool))


def _render(dev, v, f, w2c, cam):
    from xrdslam_b200.eval_recon import DepthRenderer
    r = DepthRenderer(v, f, dev, H=cam['H'], W=cam['W'], fx=cam['fx'], fy=cam['fy'],
                      cx=cam['cx'], cy=cam['cy'], near=cam['near'], far=cam['far'])
    return r.render(w2c).cpu().numpy()


SMALL = _cam(80, 96, 70.0, 64.0, 40.3, 45.7)
FULL = _cam(500, 500, 300.0, 300.0, 249.5, 249.5)


def _assert_same(got, exp):
    bad = got.view(np.uint32) != exp.view(np.uint32)
    assert not bad.any(), (bad.sum(), got[bad][:5], exp[bad][:5])


@pytest.mark.parametrize('cam,n', [(SMALL, 12), (FULL, 2)])
def test_room_depth_bit_exact_against_oracle(cuda_dev, cam, n):
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.25)
    w2c = np.linalg.inv(_views(v, n, seed=11))[:, :3]
    got = _render(cuda_dev, v, f, w2c, cam)
    _assert_same(got, ore.render_depth(v, f, w2c, cam))
    assert (got > 0).all()


@pytest.mark.parametrize('seed', [0, 1])
def test_triangle_soup_bit_exact_against_oracle(cuda_dev, seed):
    """Random triangles around the camera: many straddle the near plane or lie behind it, some
    are huge on screen (guard-band clip) and some are slivers."""
    rng = np.random.default_rng(seed)
    n = 400
    c = rng.normal(size=(n, 1, 3)) * 1.5
    v = (c + rng.normal(size=(n, 3, 3)) * rng.choice([0.02, 0.3, 3.0], size=(n, 1, 1))).reshape(-1, 3)
    v = v.astype(f32)
    f = np.arange(3 * n, dtype=np.int32).reshape(n, 3)
    from xrdslam_b200.eval_recon import viewmatrix
    c2w = np.tile(np.eye(4), (5, 1, 1))
    c2w[:, :3] = viewmatrix(rng.normal(size=(5, 3)), [0, 0, -1], rng.normal(size=(5, 3)) * 0.2)
    w2c = np.linalg.inv(c2w)[:, :3]
    for cam in (SMALL, _cam(80, 96, 70.0, 64.0, 40.3, 45.7, near=0.01, far=3.0)):
        got = _render(cuda_dev, v, f, w2c, cam)
        _assert_same(got, ore.render_depth(v, f, w2c, cam))
        assert (got > 0).mean() > 0.2


def test_no_holes_inside_the_room_at_1cm(cuda_dev):
    from xrdslam_b200.eval_recon import DepthRenderer
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.01)
    w2c = np.linalg.inv(_views(v, 64, seed=2))[:, :3]
    r = DepthRenderer(v, f, cuda_dev)
    d = r.render(w2c)
    assert int((d == 0).sum()) == 0
    n = torch.zeros(1, dtype=torch.int32, device=cuda_dev)
    from xrdslam_b200 import _cabi
    _cabi.lib().xrd_debug_eval_render_queued(r.ws.data_ptr(), n.data_ptr(), None)
    q = int(n.item())
    assert 0 < q < len(f) * min(64, r.B)  # both paths run


def test_unseen_check_matches_oracle_for_4096_candidates(cuda_dev):
    from xrdslam_b200.eval_recon import points_seen, viewmatrix
    from xrdslam_b200.synthetic import CENTRE
    rng = np.random.default_rng(5)
    a, b = np.meshgrid(np.linspace(-1.5, 0.5, 30), np.linspace(-0.5, 1.5, 30))
    pc = np.stack([np.full(a.size, 2.9), a.ravel(), b.ravel()], -1).astype(f32)
    K = 4096
    c2w = np.tile(np.eye(4), (K, 1, 1))
    o = CENTRE + rng.uniform(-1, 1, size=(K, 3))
    c2w[:, :3] = viewmatrix(rng.uniform(-1e4, 1e4, size=(K, 3)).round(2) - o, [0, 0, -1], o)
    got = points_seen(pc, c2w, device=cuda_dev)
    exp = np.array([ore.check_proj(pc, 500, 500, 300., 300., 249.5, 249.5, c) for c in c2w])
    assert np.array_equal(got, exp)
    assert 0.05 < exp.mean() < 0.95


def test_per_view_sums_bit_identical_and_equal_to_oracle(cuda_dev):
    from xrdslam_b200.eval_recon import depth_l1_sums
    rng = np.random.default_rng(2)
    gt = (rng.random((5, 97, 61)) * 4).astype(f32)
    rec = np.where(rng.random((5, 97, 61)) < 0.3, 0, rng.random((5, 97, 61)) * 4).astype(f32)
    rec[3] = 0
    g, r = torch.from_numpy(gt).to(cuda_dev), torch.from_numpy(rec).to(cuda_dev)
    a, b = depth_l1_sums(g, r).cpu().numpy(), depth_l1_sums(g, r).cpu().numpy()
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    assert np.array_equal(a.view(np.uint64), ore.depth_l1_sums(gt, rec).view(np.uint64))


def _write_room(tmp_path, spacing, pc=None):
    from xrdslam_b200 import io_formats
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(spacing)
    p = io_formats.write_ply(str(tmp_path / 'room_gt.ply'), v, f)
    if pc is None:
        a, b = np.meshgrid(np.linspace(-1.5, 0.5, 30), np.linspace(-0.5, 1.5, 30))
        pc = np.stack([np.full(a.size, 2.9), a.ravel(), b.ravel()], -1).astype(f32)
    np.save(str(tmp_path / 'room_gt_pc_unseen.npy'), pc)
    return p, v, f, pc


def test_ground_truth_against_itself_is_zero(cuda_dev, tmp_path):
    from xrdslam_b200.eval_recon import calc_2d_metric
    p, _, _, _ = _write_room(tmp_path, 0.1)
    assert calc_2d_metric(p, p, align=False, n_imgs=40, seed=1, device=cuda_dev) == \
        {'depth l1': 0.0}


def _render_args(r, w2c, depth, status, ws, nb):
    return (r.verts.data_ptr(), r.verts.shape[0], r.faces.data_ptr(), r.faces.shape[0],
            w2c.data_ptr(), w2c.shape[0], C.byref(r.camera), depth.data_ptr(), status.data_ptr(),
            ws.data_ptr(), nb, None)


@pytest.mark.parametrize('n_views', [1, 7])
def test_workspace_one_byte_short_writes_nothing(cuda_dev, n_views):
    from xrdslam_b200 import _cabi
    from xrdslam_b200.eval_recon import DepthRenderer
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.5)
    r = DepthRenderer(v, f, cuda_dev, H=40, W=50, fx=30., fy=30.)
    lib = _cabi.lib()
    nb = lib.xrd_eval_render_workspace_bytes(len(f), n_views)
    assert nb >= 4 * len(f) * n_views
    w2c = torch.from_numpy(np.linalg.inv(_views(v, n_views, 3))[:, :3].copy()).to(cuda_dev)
    depth = torch.full((n_views, 40, 50), 7.0, device=cuda_dev)
    status = torch.full((1,), 99, dtype=torch.int32, device=cuda_dev)
    ws = torch.full((nb,), 0xAB, dtype=torch.uint8, device=cuda_dev)
    assert lib.xrd_eval_render_depth(*_render_args(r, w2c, depth, status, ws, nb - 1)) == -3
    torch.cuda.synchronize()
    assert (depth == 7.0).all() and int(status.item()) == 99 and (ws == 0xAB).all()
    assert lib.xrd_eval_render_depth(*_render_args(r, w2c, depth, status, ws, nb)) == 0
    torch.cuda.synchronize()
    assert int(status.item()) == 0 and (depth > 0).all()


def test_out_of_range_faces_raise_shape(cuda_dev):
    from xrdslam_b200._cabi import XrdError
    from xrdslam_b200.eval_recon import DepthRenderer
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.5)
    for bad in (len(v), -1):
        g = f.copy()
        g[len(g) // 2, 1] = bad
        with pytest.raises(XrdError, match='XRD_E_SHAPE'):
            DepthRenderer(v, g, cuda_dev).render(np.linalg.inv(_views(v, 2, 0))[:, :3])


def _tsdf_rec(tmp_path, dev):
    import make_golden_cull as mg
    from xrdslam_b200 import io_formats
    from xrdslam_b200.common import cull_mesh, get_mesh_from_RGBD
    from xrdslam_b200.mesher import TriMesh
    from xrdslam_b200.synthetic import make_sequence

    class KF:
        def __init__(self, c2w, rgb, depth):
            self._pose, self.rgb, self.depth = torch.as_tensor(c2w), rgb, depth

        def get_pose(self):
            return self._pose

    class Algo:
        def __init__(self, gt, est):
            self.gt, self.est = gt, est

        def get_gt_c2w_list_ori(self):
            return self.gt

        def get_gt_c2w_list(self):
            return self.gt

        def get_estimate_c2w_list(self):
            return self.est

    cam, poses, frames = make_sequence(8, width=160, height=120)
    mesh = get_mesh_from_RGBD(cam, [KF(p, rgb, d) for p, (rgb, d) in zip(poses, frames)],
                              device=dev)
    host = TriMesh(mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy())
    ds = mg.Dataset(np.stack([d for _, d in frames]).astype(f32), np.stack(poses).astype(f32),
                    [cam.height, cam.width, cam.fx, cam.fy, cam.cx, cam.cy])
    cull_mesh(ds, host, None, eval_rec=True, device=dev).export(str(tmp_path / 'final_mesh_rec.ply'))
    gt = [torch.as_tensor(p) for p in poses]
    est = [g.clone() for g in gt]
    for e in est:
        e[:3, 3] += torch.tensor([0.002, -0.001, 0.0])
    io_formats.save_eval_tar(Algo(gt, est), str(tmp_path), len(gt))
    return str(tmp_path / 'final_mesh_rec.ply')


def test_calc_2d_metric_against_oracle_pipeline(cuda_dev, tmp_path):
    from xrdslam_b200 import io_formats
    from xrdslam_b200.eval_recon import (_aligned_vertices, _pts, calc_2d_metric,
                                         get_cam_position)
    rec = _tsdf_rec(tmp_path, cuda_dev)
    gt, gv, gf, pc = _write_room(tmp_path, 0.05)
    T = np.eye(4)
    T[:3, 3] = [-0.002, 0.001, 0.0]
    # two views: the numpy rasteriser takes about a minute per 500 x 500 view of both meshes
    got = calc_2d_metric(rec, gt, transform_matrix=T, n_imgs=2, seed=3, device=cuda_dev)
    rv, rf, _ = io_formats.read_ply(rec)
    rva, _ = _aligned_vertices(_pts(rv, cuda_dev), _pts(gv, cuda_dev), T, True, 30)
    rva = rva.cpu().numpy()
    ext, tr = get_cam_position(gv)
    c2w = ore.sample_views_sequential(pc, ext, tr, 2, seed=3)
    w2c = np.linalg.inv(c2w)[:, :3]
    near = lambda x: 0.01 * float(np.max(x.max(0) - x.min(0)))
    gd = ore.render_depth(gv, gf, w2c, _cam(500, 500, 300., 300., 249.5, 249.5, near(gv)))
    rd = ore.render_depth(rva, rf, w2c, _cam(500, 500, 300., 300., 249.5, 249.5, near(rva)))
    s = ore.depth_l1_sums(gd, rd)
    ok = s[:, 1] > 0
    exp = (s[ok, 0] / s[ok, 1]).mean() * 100
    assert abs(got['depth l1'] - exp) <= 1e-9 * exp, (got, exp)
    assert np.isfinite(exp) and exp > 0


def test_eval_matrics_with_depth_l1_end_to_end(cuda_dev, tmp_path):
    from xrdslam_b200.eval import EvalMatrics
    from xrdslam_b200.eval_recon import calc_2d_metric
    _tsdf_rec(tmp_path, cuda_dev)
    gt, _, _, _ = _write_room(tmp_path, 0.05)
    m = EvalMatrics(output_dir=tmp_path, gt_mesh=gt, seed=4, eval_2d_metric=True)
    res = m.main()
    assert next(iter(res)) == 'depth l1'
    d = res['depth l1']
    # 8 frames over a quarter turn reconstruct part of the room: views that see the
    # reconstruction's walls where the ground truth has a nearer box or wall add centimetres
    assert np.isfinite(d) and 0 < d < 5
    _, T = m.trajectory()
    assert calc_2d_metric(str(tmp_path / 'final_mesh_rec.ply'), gt, transform_matrix=T,
                          seed=4, device=cuda_dev)['depth l1'] == d
    off = EvalMatrics(output_dir=tmp_path, gt_mesh=gt, seed=4).main()
    assert {k: v for k, v in res.items() if k != 'depth l1'} == off
