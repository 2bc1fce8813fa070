"""cull_mesh on the device (csrc/cull.cu, common.cull_mesh): bit for bit against the numpy
restatement (oracle/cull.py (a)); against the reference's decisions (the golden fixture) and the
reference's torch loop run on this GPU ((b)) under the borderline rule; and
Algorithm.save_final_mesh end to end."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import cull as oc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_cull as mg  # noqa: E402
from test_cull_cpu import GOLDEN, analytic_cases, borderline_check  # noqa: E402

pytestmark = pytest.mark.gpu
f32 = np.float32


def _camera_row(cam):
    return [cam.height, cam.width, cam.fx, cam.fy, cam.cx, cam.cy]


def _room_mesh(dev, depth, poses, cam, n_random=20000, seed=0):
    """The TSDF mesh of the frames (get_mesh_from_RGBD's volume) plus seeded random vertices in
    and around the room box, with random faces over them and uint8 colours: host arrays."""
    from xrdslam_b200.synthetic import ROOM
    from xrdslam_b200.tsdf import TSDFVolume, o3d_poses
    c2w, w2c = o3d_poses(poses)
    vol = TSDFVolume(device=dev)
    color = torch.full(depth.shape + (3, ), 128, dtype=torch.uint8, device=dev)
    vol.integrate(torch.from_numpy(depth).to(dev), color, c2w, (cam.fx, cam.fy, cam.cx, cam.cy),
                  w2c=w2c)
    v, f, _ = vol.extract_triangle_mesh()
    v, f = v.cpu().numpy(), f.cpu().numpy()
    rng = np.random.default_rng(seed)
    rv = rng.uniform(ROOM[:, 0] - 0.5, ROOM[:, 1] + 0.5, (n_random, 3)).astype(f32)
    rf = (rng.integers(0, n_random, (n_random, 3)) + v.shape[0]).astype(np.int32)
    verts = np.concatenate([v, rv])
    faces = np.concatenate([f, rf])
    colors = rng.integers(0, 256, (verts.shape[0], 3)).astype(np.uint8)
    return verts, faces, colors


def _sequence(n, width, height):
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(n, width=width, height=height)
    depth = np.stack([d for _, d in frames]).astype(f32)
    return cam, np.stack(poses).astype(f32), depth


def _w2c_used(dev, poses):
    return np.stack([torch.inverse(torch.as_tensor(p).to(dev).float())[:3].cpu().numpy()
                     for p in poses])


def _check(dev, ds, depth, verts, faces, colors, est, eval_rec, trunc, chunk, label):
    """CUDA == (a) bit for bit (seen, vertices, faces, colours); CUDA vs (b) on this GPU under
    the borderline rule.  -> the culled TriMesh."""
    from xrdslam_b200.common import cull_mesh, cull_visibility
    from xrdslam_b200.mesher import TriMesh
    n = len(est) if est is not None else len(ds)
    poses = [est[i] if est is not None else ds[i][3] for i in range(n)]
    w2c = _w2c_used(dev, poses)
    seen = cull_visibility(ds, torch.from_numpy(verts).to(dev), est, eval_rec, trunc, dev,
                           chunk).cpu().numpy().astype(bool)
    seen_a = oc.visible(verts, w2c, depth[:n], ds.get_camera(), trunc, eval_rec)
    assert np.array_equal(seen, seen_a)
    assert 0 < seen.sum()
    mesh = cull_mesh(ds, TriMesh(verts, faces, colors), est, eval_rec, trunc, dev, chunk)
    v, f, c = oc.compact(seen_a, verts, faces, colors)
    assert np.array_equal(mesh.vertices.view(np.uint32), v.view(np.uint32))
    assert np.array_equal(mesh.faces, f) and mesh.faces.dtype == np.int32
    assert np.array_equal(mesh.vertex_colors, c)
    seen_b = oc.reference_seen(ds, verts, est, eval_rec, trunc, device=dev).cpu().numpy()
    nb = borderline_check(seen, seen_b, verts, w2c, depth[:n], ds.get_camera(), trunc, eval_rec)
    print(f'{label}: V={verts.shape[0]} seen={int(seen.sum())} kept F={f.shape[0]} of '
          f'{faces.shape[0]}; {nb} borderline disagreements with the torch loop on the GPU')
    return mesh


def test_w2c_is_torch_inverse_bit_for_bit(cuda_dev):
    from xrdslam_b200.common import cull_w2c
    _, poses, _ = _sequence(8, 64, 48)
    buf = torch.from_numpy(poses).to(cuda_dev)
    for k in range(len(poses)):
        ref = torch.inverse(torch.from_numpy(poses[k]).to(cuda_dev))[:3]
        assert torch.equal(cull_w2c(buf[k]).view(torch.int32), ref.contiguous().view(torch.int32))


# (size, frames, chunk, estimate poses: None / 'all' / 'short', eval_rec, truncation)
SEQ_CASES = [
    ((160, 120), 7, 3, None, True, 0.06),
    ((160, 120), 6, 1, 'short', True, 0.06),
    ((160, 120), 5, 16, 'all', False, 0.06),
    ((160, 120), 7, 4, None, True, 0.02),
    ((640, 480), 5, 2, 'all', True, 0.06),
    ((640, 480), 4, 3, 'short', False, 0.06),
]


@pytest.mark.parametrize('size,n,chunk,est_mode,eval_rec,trunc', SEQ_CASES)
def test_sequence_matches_restatement(cuda_dev, size, n, chunk, est_mode, eval_rec, trunc):
    cam, poses, depth = _sequence(n, *size)
    verts, faces, colors = _room_mesh(cuda_dev, depth, poses, cam)
    ds = mg.Dataset(depth, poses, _camera_row(cam))
    est = None
    if est_mode is not None:
        rng = np.random.default_rng(1)
        e = poses.copy()
        e[:, :3, 3] += rng.normal(0, 0.02, (n, 3)).astype(f32)
        est = [torch.from_numpy(p) for p in (e if est_mode == 'all' else e[:-2])]
    _check(cuda_dev, ds, depth, verts, faces, colors, est, eval_rec, trunc, chunk,
           f'{size} n={n} chunk={chunk} est={est_mode} rec={eval_rec} t={trunc}')


def test_back_to_back_calls_without_a_host_sync(cuda_dev):
    """cull_visibility is asynchronous on the caller's stream: a second call, enqueued while the
    first call's launches may still run, must not upload into memory they read."""
    from xrdslam_b200.common import cull_visibility
    cam, poses, depth = _sequence(12, 640, 480)
    verts, _, _ = _room_mesh(cuda_dev, depth[:3], poses[:3], cam, n_random=200000)
    vd = torch.from_numpy(verts).to(cuda_dev)
    other = np.ascontiguousarray(depth[::-1] * f32(0.5))
    other_poses = np.ascontiguousarray(poses[::-1])
    torch.cuda.synchronize()
    s1 = cull_visibility(mg.Dataset(depth, poses, _camera_row(cam)), vd, None, True, 0.06,
                         cuda_dev, 4)
    s2 = cull_visibility(mg.Dataset(other, other_poses, _camera_row(cam)), vd, None, True, 0.06,
                         cuda_dev, 4)
    e1 = oc.visible(verts, _w2c_used(cuda_dev, poses), depth, cam, 0.06, True)
    e2 = oc.visible(verts, _w2c_used(cuda_dev, other_poses), other, cam, 0.06, True)
    assert (e1 != e2).sum() > 1000
    assert np.array_equal(s1.cpu().numpy().astype(bool), e1)
    assert np.array_equal(s2.cpu().numpy().astype(bool), e2)


@pytest.mark.parametrize('name,use_est,eval_rec,trunc', mg.CASES)
def test_golden_reference_decisions(cuda_dev, name, use_est, eval_rec, trunc):
    from xrdslam_b200.common import cull_visibility
    g = dict(np.load(GOLDEN))
    ds = mg.Dataset(g['depth'], g['poses'], g['camera'])
    est = [torch.from_numpy(p) for p in g['est']] if use_est else None
    poses = g['est'] if use_est else g['poses']
    w2c = _w2c_used(cuda_dev, poses)
    seen = cull_visibility(ds, torch.from_numpy(g['verts']).to(cuda_dev), est, eval_rec, trunc,
                           cuda_dev, 2).cpu().numpy().astype(bool)
    assert np.array_equal(seen, oc.visible(g['verts'], w2c, g['depth'][:len(poses)], ds.cam, trunc,
                                           eval_rec))
    nb = borderline_check(seen, g[name + '_seen'], g['verts'], w2c, g['depth'][:len(poses)],
                          ds.cam, trunc, eval_rec)
    # kept faces differ only where a face holds a (borderline) disagreeing vertex
    kept = seen[g['faces']].any(1)
    near = (seen != g[name + '_seen'])[g['faces']].any(1)
    assert not ((kept != g[name + '_kept']) & ~near).any()
    print(f'golden {name}: {nb} borderline disagreements with the reference of {seen.size}')


def test_host_and_device_inputs_give_identical_output(cuda_dev):
    from xrdslam_b200.common import cull_mesh
    from xrdslam_b200.mesher import TriMesh
    cam, poses, depth = _sequence(5, 160, 120)
    verts, faces, colors = _room_mesh(cuda_dev, depth, poses, cam, n_random=5000)
    est = [torch.from_numpy(p) for p in poses[:4]]
    host = cull_mesh(mg.Dataset(depth, poses, _camera_row(cam)), TriMesh(verts, faces, colors),
                     est, True, device=cuda_dev, chunk=3)
    dmesh = TriMesh(torch.from_numpy(verts).to(cuda_dev), torch.from_numpy(faces).to(cuda_dev),
                    torch.from_numpy(colors).to(cuda_dev))
    fcol = TriMesh(verts, faces, colors.astype(f32) / 255)          # float colours carried too
    dev = cull_mesh(mg.Dataset(depth, poses, _camera_row(cam), device=cuda_dev), dmesh,
                    [p.to(cuda_dev) for p in est], True, device=cuda_dev, chunk=3)
    fc = cull_mesh(mg.Dataset(depth, poses, _camera_row(cam)), fcol, est, True, device=cuda_dev)
    assert host.faces.shape[0] > 1000
    for a in (dev, fc):
        assert np.array_equal(a.vertices.view(np.uint32), host.vertices.view(np.uint32))
        assert np.array_equal(a.faces, host.faces)
    assert np.array_equal(dev.vertex_colors, host.vertex_colors)
    assert fc.vertex_colors.dtype == np.float32
    assert np.array_equal(fc.vertex_colors, host.vertex_colors.astype(f32) / 255)
    none = cull_mesh(mg.Dataset(depth, poses, _camera_row(cam)), TriMesh(verts, faces), est,
                     True, device=cuda_dev)
    assert none.vertex_colors is None and np.array_equal(none.faces, host.faces)


@pytest.mark.parametrize('case', analytic_cases(), ids=lambda c: c[0])
def test_analytic_visibility(cuda_dev, case):
    from xrdslam_b200.common import cull_visibility
    _, verts, cam, depth, eval_rec, trunc, expect = case
    ds = mg.Dataset(np.asarray(depth, f32)[None], np.eye(4, dtype=f32)[None], _camera_row(cam))
    seen = cull_visibility(ds, torch.tensor(verts, dtype=torch.float32), None, eval_rec, trunc,
                           cuda_dev)
    assert seen.bool().cpu().tolist() == expect


def test_nothing_and_everything_visible(cuda_dev):
    from xrdslam_b200.common import cull_mesh
    from xrdslam_b200.mesher import TriMesh
    cam = type('Cam', (), dict(width=16, height=12, fx=10.0, fy=10.0, cx=8.0, cy=6.0))
    rng = np.random.default_rng(0)
    front = np.concatenate([rng.uniform(-0.2, 0.2, (300, 2)), rng.uniform(-1.5, -0.5, (300, 1))],
                           1).astype(f32)
    faces = rng.integers(0, 300, (500, 3)).astype(np.int32)
    colors = rng.integers(0, 256, (300, 3)).astype(np.uint8)
    ds = mg.Dataset(np.full((3, 12, 16), 2.0, f32), np.repeat(np.eye(4, dtype=f32)[None], 3, 0),
                    _camera_row(cam))
    used = np.unique(faces)
    out = cull_mesh(ds, TriMesh(front, faces, colors), eval_rec=True, device=cuda_dev)
    v, f, c = oc.compact(np.ones(300, bool), front, faces, colors)
    assert out.vertices.shape[0] == used.size
    assert np.array_equal(out.vertices, front[used]) and np.array_equal(out.faces, f)
    assert np.array_equal(out.vertex_colors, c)
    behind = front * np.array([1, 1, -1], f32)
    out = cull_mesh(ds, TriMesh(behind, faces, colors), eval_rec=True, device=cuda_dev)
    assert out.vertices.shape == (0, 3) and out.faces.shape == (0, 3)
    assert out.vertex_colors.shape == (0, 3)
    empty = cull_mesh(ds, TriMesh(np.zeros((0, 3), f32), np.zeros((0, 3), np.int32)),
                      device=cuda_dev)
    assert empty.vertices.shape == (0, 3) and empty.faces.shape == (0, 3)
    with pytest.raises(ValueError):
        cull_mesh(ds, TriMesh(front, np.array([[0, 1, 300]], np.int32)), device=cuda_dev)


# ---- Algorithm.save_final_mesh -----------------------------------------------------------------
def test_save_final_mesh_end_to_end(cuda_dev, tmp_path):
    from test_tsdf_gpu import _point_slam
    from xrdslam_b200 import io_formats
    from xrdslam_b200.common import cull_mesh
    algo, cam, fr, losses = _point_slam(cuda_dev, n_frames=3)
    assert algo.save_final_mesh(str(tmp_path / 'none'), None) is None   # no keyframe yet
    for k in range(2):
        algo.add_keyframe(fr[k])
        losses(algo, [fr[k]], 4, True)
        algo.set_initialized()
    for f in fr:
        pose = f.get_pose().detach()
        algo.add_framepose(pose, pose, pose)
    depth = np.stack([np.asarray(f.depth, f32) for f in fr])
    gt = np.stack([f.get_pose().detach().cpu().numpy() for f in fr]).astype(f32)
    ds = mg.Dataset(depth, gt, _camera_row(cam))
    paths = algo.save_final_mesh(str(tmp_path), ds)
    assert [os.path.basename(p) for p in paths] == ['final_mesh.ply', 'final_mesh_rec.ply']
    mesh = algo.get_mesh()
    v0, f0, c0 = io_formats.read_ply(paths[0])
    assert np.array_equal(v0, mesh.vertices) and np.array_equal(f0, mesh.faces)
    exp = cull_mesh(ds, mesh, algo.get_estimate_c2w_list(), eval_rec=True, device=cuda_dev)
    v1, f1, c1 = io_formats.read_ply(paths[1])
    assert v1.shape == exp.vertices.shape and f1.shape == exp.faces.shape
    assert np.array_equal(v1, exp.vertices) and np.array_equal(f1, exp.faces)
    assert np.array_equal(c1, exp.vertex_colors)
    assert 0 < f1.shape[0] <= f0.shape[0]
    print(f'save_final_mesh: final_mesh {v0.shape[0]} / {f0.shape[0]}, final_mesh_rec '
          f'{v1.shape[0]} / {f1.shape[0]}')
