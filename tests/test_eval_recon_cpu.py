"""ds-eval reconstruction metrics without a GPU: the numpy restatement (oracle/eval_recon.py)
against scipy's cKDTree and analytic cases, the sample-count rule, oracle ICP, read_ply's new
property and index types, and EvalMatrics' host-only part."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_recon as oe

f32 = np.float32


def _lattice(n=60, spacing=0.01, z=0.0):
    a, b = np.meshgrid(np.arange(n) * spacing, np.arange(n) * spacing, indexing='ij')
    return np.stack([a.ravel(), b.ravel(), np.full(a.size, z)], 1).astype(f32)


def test_brute_force_agrees_with_ckdtree_within_1e5():
    rng = np.random.default_rng(0)
    P = rng.uniform(-20, 20, (4000, 3)).astype(f32)
    Q = rng.uniform(-20, 20, (3000, 3)).astype(f32)
    d, i = oe.nn_brute(Q, P)
    d64, _ = oe.ckdtree_dist(Q, P)
    assert np.abs(d.astype(np.float64) - d64).max() <= 1e-5
    for tau in (0.5, 1.0, 2.0):
        differ = (d < f32(tau)) != (d64 < tau)
        assert np.all(np.abs(d64[differ] - tau) <= 1e-5)


def test_planar_lattices_offset_along_the_normal():
    delta = 0.03
    gt, rec = _lattice(), _lattice(z=delta)
    m = oe.calc_3d_from_points(rec, gt)
    assert abs(m['accuracy'] / 100 - delta) < 1e-6 and abs(m['completion'] / 100 - delta) < 1e-6
    assert m['completion ratio'] == 100.0
    d1, _ = oe.nn_brute(rec, gt)
    d2, _ = oe.nn_brute(gt, rec)
    h = oe.fscore_assembly(d1, d2, 0.01)
    assert h['precision'] == 0 and h['recall'] == 0 and h['fscore'] == 0
    assert abs(h['mean1'] - delta) < 1e-6 and abs(h['mean2'] - delta) < 1e-6


def test_self_query_gives_zero_and_own_id_smallest_at_duplicates():
    rng = np.random.default_rng(1)
    P = rng.uniform(-1, 1, (2000, 3)).astype(f32)
    P[1500:1600] = P[100:200]    # duplicates of earlier points
    d, i = oe.nn_brute(P, P)
    assert np.all(d == 0)
    exp = np.arange(len(P))
    exp[1500:1600] = np.arange(100, 200)
    assert np.array_equal(i, exp)


def test_radius_bound_is_inclusive():
    P = np.array([[0.1, 0, 0], [0, 0.2, 0]], f32)
    Q = np.array([[0, 0, 0], [0, 0.35, 0]], f32)
    d, i = oe.nn_brute(Q, P, radius=0.1)
    assert i[0] == 0 and d[0] == np.sqrt(f32(0.1) * f32(0.1)) and i[1] == -1 and np.isinf(d[1])


def test_reduction_order_restatement_is_a_sum():
    rng = np.random.default_rng(2)
    x = rng.random((10001, 3))
    assert np.allclose(oe.reduce_f64(x), x.sum(0), rtol=1e-13)


@pytest.mark.parametrize('gt_fewer', [True, False])
def test_sample_count_rule_takes_both_branches(gt_fewer):
    from xrdslam_b200.synthetic import room_mesh
    gv, gf = room_mesh(0.5 if gt_fewer else 0.25)
    rv, rf = room_mesh(0.25 if gt_fewer else 0.5)
    res = oe.ds_eval_3d(rv, rf, gv, gf, np.eye(4), tau=0.3, n_samples=2000, nn=oe.nn_brute)
    assert res['precision'] > 0.9 and res['recall'] > 0.9
    assert (len(gv) < len(rv)) == gt_fewer


def test_samplers_follow_the_rules():
    from xrdslam_b200.synthetic import room_mesh
    v, f = room_mesh(0.5)
    U = oe.philox_uniforms(3, 5000, 3)
    p, fi = oe.sample_trimesh(v, f, U)
    cum, tot = oe.area_prefix(v, f)
    assert np.all(cum[fi] >= U[:, 0].astype(np.float64) * tot)
    p2, fi2 = oe.sample_open3d(v, f, 5000, U[:, :2])
    assert np.all(np.diff(fi2) >= 0) and len(fi2) == 5000     # deterministic, ordered faces
    for pts in (p, p2):
        lo, hi = v.min(0) - 1e-6, v.max(0) + 1e-6
        assert np.all((pts >= lo) & (pts <= hi))


def _rot(deg, axis):
    a = np.deg2rad(deg)
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def test_oracle_icp_recovers_a_rigid_motion():
    from xrdslam_b200.synthetic import room_mesh
    gv, _ = room_mesh(0.25)
    T = np.eye(4)
    T[:3, :3] = _rot(2.0, [0.3, -0.5, 1.0])
    T[:3, 3] = [0.03, -0.01, 0.02]
    src = oe.transform(gv, np.linalg.inv(T))
    r = oe.registration_icp(src, gv, 0.1, max_iteration=50)
    assert np.abs(r['transformation'] - T).max() < 1e-4
    assert r['iterations'] < 50 and r['fitness'] > 0.99
    r1 = oe.registration_icp(src, gv, 0.1, max_iteration=1)
    assert r1['iterations'] == 1


def _write_custom_ply(path, verts, faces, vtypes, count_t, index_t, extra_face_prop=False):
    tmap = {'float': '<f4', 'double': '<f8', 'int': '<i4', 'uint': '<u4', 'short': '<i2',
            'ushort': '<u2', 'char': 'i1', 'uchar': 'u1'}
    hdr = ['ply', 'format binary_little_endian 1.0', 'comment test', f'element vertex {len(verts)}']
    hdr += [f'property {t} {n}' for n, t in zip(('x', 'y', 'z'), vtypes)]
    hdr += ['property ushort quality', 'property uchar red', 'property uchar green',
            'property uchar blue', f'element face {len(faces)}']
    hdr += [f'property list {count_t} {index_t} vertex_indices']
    if extra_face_prop:
        hdr += ['property int flags']
    vdt = np.dtype([(n, tmap[t]) for n, t in zip(('x', 'y', 'z'), vtypes)] +
                   [('q', '<u2'), ('r', 'u1'), ('g', 'u1'), ('b', 'u1')])
    rec = np.zeros(len(verts), vdt)
    rec['x'], rec['y'], rec['z'] = verts[:, 0], verts[:, 1], verts[:, 2]
    rec['r'] = 7
    fdt = [('n', tmap[count_t]), ('i', tmap[index_t], (3,))] + ([('fl', '<i4')] if extra_face_prop
                                                                 else [])
    fr = np.zeros(len(faces), np.dtype(fdt))
    fr['n'] = 3
    fr['i'] = faces
    with open(path, 'wb') as fh:
        fh.write(('\n'.join(hdr) + '\nend_header\n').encode())
        fh.write(rec.tobytes())
        fh.write(fr.tobytes())


@pytest.mark.parametrize('vtypes,count_t,index_t,extra', [
    (('float', 'float', 'float'), 'uchar', 'int', False),
    (('double', 'double', 'double'), 'ushort', 'uint', True),
    (('int', 'short', 'char'), 'int', 'int', False),
    (('uint', 'ushort', 'uchar'), 'uint', 'uint', True),
])
def test_read_ply_property_and_index_types(tmp_path, vtypes, count_t, index_t, extra):
    from xrdslam_b200.io_formats import read_ply
    verts = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9], [10, 11, 12]], np.float64)
    faces = np.array([[0, 1, 2], [1, 2, 3]])
    p = str(tmp_path / 'm.ply')
    _write_custom_ply(p, verts, faces, vtypes, count_t, index_t, extra)
    v, f, c = read_ply(p)
    assert v.dtype == np.float32 and np.array_equal(v, verts.astype(f32))
    assert f.dtype == np.int32 and np.array_equal(f, faces)
    assert np.all(c[:, 0] == 7)


def test_read_ply_rejects_ascii_and_big_endian(tmp_path):
    from xrdslam_b200.io_formats import read_ply
    for fmt in ('ascii', 'binary_big_endian'):
        p = tmp_path / f'{fmt}.ply'
        p.write_bytes(f'ply\nformat {fmt} 1.0\nelement vertex 0\nproperty float x\n'
                      'end_header\n'.encode())
        with pytest.raises(ValueError, match='binary_little_endian'):
            read_ply(str(p))


def test_read_ply_round_trips_unchanged(tmp_path):
    from xrdslam_b200.io_formats import read_ply, write_ply
    rng = np.random.default_rng(3)
    v = rng.random((50, 3)).astype(f32)
    f = rng.integers(0, 50, (30, 3)).astype(np.int32)
    c = rng.integers(0, 256, (50, 3)).astype(np.uint8)
    for faces, colors in ((f, c), (f, None), (None, c), (None, None)):
        v2, f2, c2 = read_ply(write_ply(str(tmp_path / 'r.ply'), v, faces, colors))
        assert np.array_equal(v2, v)
        assert (f2 is None) if faces is None else np.array_equal(f2, faces)
        assert (c2 is None) if colors is None else np.array_equal(c2, colors)


class _Algo:
    def __init__(self, gt, est):
        self.gt, self.est = gt, est

    def get_gt_c2w_list_ori(self):
        return self.gt

    def get_gt_c2w_list(self):
        return self.gt

    def get_estimate_c2w_list(self):
        return self.est


def test_eval_matrics_host_part_to_the_first_device_call(tmp_path, monkeypatch):
    from xrdslam_b200 import eval as ev
    from xrdslam_b200.io_formats import save_eval_tar, write_ply
    from xrdslam_b200.synthetic import room_mesh, trajectory
    gt = [torch.as_tensor(p) for p in trajectory(6)]
    est = [g.clone() for g in gt]
    for e in est:
        e[:3, 3] += 0.01
    save_eval_tar(_Algo(gt, est), str(tmp_path), 6)
    v, f = room_mesh(0.5)
    write_ply(str(tmp_path / 'final_mesh_rec.ply'), v, f)
    gt_path = write_ply(str(tmp_path / 'room.ply'), v, f)
    calls = []

    def first_device_call(rec, gtm, transform_matrix=None, **kw):
        calls.append(transform_matrix)
        raise RuntimeError('device')

    import xrdslam_b200.eval_recon as er
    monkeypatch.setattr(er, 'calc_3d_metric', first_device_call)
    m = ev.EvalMatrics(output_dir=tmp_path, gt_mesh=gt_path)
    with pytest.raises(RuntimeError, match='device'):
        m.main()
    assert abs(m.traj_result['rmse']) < 1e-6
    T = calls[0]
    assert T.shape == (4, 4) and np.allclose(T[:3, 3], -0.01, atol=1e-6)
    with pytest.raises(NotImplementedError, match='depth renderer'):
        ev.EvalMatrics(output_dir=tmp_path, gt_mesh=gt_path, eval_2d_metric=True).main()
    assert ev.EvalMatrics(output_dir=tmp_path / 'missing', gt_mesh=gt_path).main() is None
    with pytest.raises(RuntimeError, match='device'):
        ev.entrypoint(['--output_dir', str(tmp_path), '--gt_mesh', gt_path])
    assert os.path.exists(tmp_path / 'eval.tar')
