"""Marching cubes without a GPU: the generated case table, the numpy restatement of the CUDA
kernels (oracle/marching_cubes.py) on analytic fields, and the Mesher's lattice / bound mask
against the reference's own Mesher."""
import os

import numpy as np
import pytest
import torch

from oracle import marching_cubes as mc
from oracle import mc_table

f32 = np.float32


def test_committed_table_matches_generator():
    with open(mc_table.HEADER) as f:
        assert f.read() == mc_table.render_header()
    assert mc_table.max_triangles() == mc.MAX_TRI == 5


def test_case_triangles_use_exactly_the_crossed_edges():
    tables = mc_table.build()
    for case in range(256):
        crossed = {e for e in range(12) if mc_table._crossed(case, e)}
        used = {e for t in tables[case] for e in t}
        assert used == crossed, case
        for t in tables[case]:
            assert len(set(t)) == 3


def _lattice(n=(34, 30, 38), lo=-1.0, hi=1.0):
    axes = [np.linspace(lo, hi, k) for k in n]
    X, Y, Z = np.meshgrid(*axes, indexing='ij')
    sp = [a[1] - a[0] for a in axes]
    return X, Y, Z, sp, [a[0] for a in axes]


def _sphere(X, Y, Z, r=0.6, c=(0.05, -0.03, 0.02)):
    return np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r


def _torus(X, Y, Z, R=0.55, r=0.22):
    return np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R) ** 2 + Z ** 2) - r


def _two_spheres(X, Y, Z):
    return np.minimum(_sphere(X, Y, Z, 0.35, (-0.45, 0, 0)), _sphere(X, Y, Z, 0.3, (0.5, 0.1, 0)))


def _random_smooth(seed, shape=(26, 21, 30), quantise=False):
    """Sum of random Gaussian bumps below a threshold, positive on the border."""
    rng = np.random.default_rng(seed)
    X, Y, Z, _, _ = _lattice(shape)
    f = np.full(X.shape, 0.4)
    for _ in range(8):
        c = rng.uniform(-0.7, 0.7, 3)
        s = rng.uniform(0.15, 0.4)
        f -= rng.uniform(0.3, 1.0) * np.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) / s ** 2)
    if quantise:  # many lattice values exactly at the level
        f = np.round(f * 8) / 8
    f[[0, -1]] = f[:, [0, -1]] = f[:, :, [0, -1]] = 1.0
    return f.astype(f32)


def _closed_oriented(faces):
    und, di = mc.edge_use(faces)
    assert set(und.values()) == {2}      # every undirected edge in exactly two faces
    assert set(di.values()) == {1}       # every directed edge once: consistent winding


@pytest.mark.parametrize('field,chi', [(_sphere, 2), (_torus, 0), (_two_spheres, 4)])
def test_analytic_fields_closed_oriented(field, chi):
    X, Y, Z, sp, o = _lattice()
    v, f = mc.marching_cubes(field(X, Y, Z).astype(f32)[None], 0.0, sp, o)
    assert f.shape[0] > 100
    _closed_oriented(f)
    assert mc.euler_characteristic(v, f) == chi
    assert np.unique(f).size == v.shape[0]  # every vertex is used


def test_sphere_volume_and_outward_winding():
    X, Y, Z, sp, o = _lattice((60, 56, 64))
    r = 0.6
    v, f = mc.marching_cubes(_sphere(X, Y, Z, r).astype(f32)[None], 0.0, sp, o)
    vol = mc.signed_volume(v, f)
    assert vol > 0  # normals point toward larger values = outward
    assert abs(vol / (4.0 / 3.0 * np.pi * r ** 3) - 1) < 0.01


@pytest.mark.parametrize('seed,quantise', [(0, False), (1, False), (2, True), (3, True)])
def test_random_smooth_fields_closed_oriented(seed, quantise):
    f = _random_smooth(seed, quantise=quantise)
    assert (f < 0).any()
    v, fc = mc.marching_cubes(f[None], 0.0, (0.1, 0.2, 0.3))
    _closed_oriented(fc)


def _vertices_by_loop(values, level, spacing, shift, scale, origin):
    """Plain loops over (volume, lattice index, axis): the fp32 interpolation on every crossed
    lattice edge, in the documented vertex order."""
    B, nx, ny, nz = values.shape
    lev = f32(level)
    out = []
    for b in range(B):
        for i in range(nx):
            for j in range(ny):
                for k in range(nz):
                    v0 = values[b, i, j, k]
                    for a, (di, dj, dk) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
                        if i + di >= nx or j + dj >= ny or k + dk >= nz:
                            continue
                        v1 = values[b, i + di, j + dj, k + dk]
                        if (v0 < lev) == (v1 < lev):
                            continue
                        t = f32(f32(lev - v0) / f32(v1 - v0))
                        p = [f32(i), f32(j), f32(k)]
                        p[a] = f32(p[a] + t)
                        out.append([f32(f32(f32(f32(p[d] * f32(spacing[d])) + f32(shift[d])) *
                                                f32(scale[d])) + f32(origin[b][d]))
                                    for d in range(3)])
    return np.array(out, f32).reshape(-1, 3)


def test_vertices_are_fp32_edge_interpolations_in_order():
    rng = np.random.default_rng(5)
    vals = rng.standard_normal((3, 5, 4, 6)).astype(f32)
    vals[0, 1, 1, 1] = 0.0  # exactly at the level: positive side
    origin = rng.standard_normal((3, 3)).astype(f32)
    sp, sh, sc = (1 / 7, 1 / 7, 1 / 7), (-0.5,) * 3, (0.2,) * 3
    v, f = mc.marching_cubes(vals, 0.0, sp, sh, sc, origin)
    ref = _vertices_by_loop(vals, 0.0, sp, sh, sc, origin)
    assert np.array_equal(v.view(np.uint32), ref.view(np.uint32))
    # every face lies in one volume and references existing vertices
    per_volume = np.cumsum([0] + [len(_vertices_by_loop(vals[b:b + 1], 0.0, sp, sh, sc, origin[b:b + 1]))
                                  for b in range(3)])
    vol_of = np.searchsorted(per_volume, f, side='right') - 1
    assert (vol_of == vol_of[:, :1]).all() and f.max() < v.shape[0]


def test_no_crossing_gives_empty_mesh():
    for val in (1.0, -1.0, 0.0):
        v, f = mc.marching_cubes(np.full((2, 4, 5, 6), val, f32), 0.0, (1, 1, 1))
        assert v.shape == (0, 3) and f.shape == (0, 3)


# ---- the Mesher's lattice, point order and bound mask vs the reference's own Mesher ------
@pytest.mark.needs_reference
def test_mesher_grid_and_mask_match_reference():
    from oracle import ref_harness
    ref_harness.install()
    from slam.common.mesher import Mesher as RefMesher
    from slam.common.mesher import MesherConfig as RefMesherConfig
    from xrdslam_b200.mesher import Mesher, MesherConfig
    mc_bound = torch.from_numpy(np.array([[-2.2, 2.6], [-3.4, 2.1], [-1.4, 2.0]]))
    bbox = torch.from_numpy(np.array([[-2.0, 2.2], [-3.4, 1.7], [-1.25, 1.6]]))
    res, bs = 23, 1000
    ref = RefMesher(RefMesherConfig(resolution=res, points_batch_size=bs), None, bbox, mc_bound)
    own = Mesher(MesherConfig(resolution=res, points_batch_size=bs), None, bbox, mc_bound)
    g_ref = ref.get_grid_uniform(res)
    xyz = own.get_grid_uniform(res)['xyz']
    for a, b in zip(xyz, g_ref['xyz']):
        assert np.array_equal(a, np.asarray(b))
    n = res ** 3
    pts = own.grid_points(xyz, 0, n, 'cpu')
    # reference order: meshgrid 'xy' (y slowest); the volume is its transpose [1, 0, 2]
    ref_pts = g_ref['grid_points'].reshape(res, res, res, 3).transpose(0, 1).reshape(-1, 3)
    assert torch.equal(pts, ref_pts)
    # chunked generation gives the same points
    assert torch.equal(torch.cat([own.grid_points(xyz, s, min(777, n - s), 'cpu')
                                  for s in range(0, n, 777)]), pts)
    fn = lambda p: p[:, :1].clone() * 0 + 1
    got = own.eval_points(pts, fn, bbox)
    exp = ref.eval_points(pts, fn, bbox)
    assert torch.equal(got, exp) and (got == 100).any() and (got == 1).any()
    # the vertex colour path passes float32 points of arbitrary position
    g = torch.Generator().manual_seed(0)
    q = (torch.rand(5000, 3, generator=g) * 6 - 3).float()
    q[:50, 0] = float(bbox[0][0])  # exactly on the bound (float32 of the float64 bound)
    fn3 = lambda p: torch.ones(p.shape[0], 1, 3)
    assert torch.equal(own.eval_points(q, fn3, bbox), ref.eval_points(q, fn3, bbox))
