"""The numpy restatement of the TSDF fusion, its marching cubes and clean_mesh (oracle/tsdf.py)
on the CPU: allocation against a brute-force set, a fronto-parallel plane against the analytic
TSDF, mesh topology and geometry on the synthetic room, components against scipy."""
import numpy as np
import pytest

from oracle import tsdf as ot
from oracle.marching_cubes import edge_use

f32 = np.float32


def _room(n, width=160, height=120):
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(n, width=width, height=height)
    c2w, w2c = ot.o3d_poses(poses)
    depth = np.stack([d for _, d in frames])
    color = np.stack([(rgb * 255).astype(np.uint8) for rgb, _ in frames])
    return cam, poses, depth, color, c2w, w2c


def test_allocation_equals_brute_force_set():
    cam, _, depth, _, c2w, _ = _room(3)
    P = ot.Params(cam)
    keys, masks = ot.allocate(depth, c2w, P)
    assert np.all(np.diff(keys) > 0)
    for k in range(depth.shape[0]):
        want = set()
        T = c2w[k]
        for v in range(0, cam.height, 4):
            for u in range(0, cam.width, 4):
                d = f32(depth[k, v, u])
                if not d > 0:
                    continue
                x = ((f32(u) - P.cx) * d) / P.fx
                y = ((f32(v) - P.cy) * d) / P.fy
                lo, hi = [], []
                for a in range(3):
                    p = ((T[a, 0] * x + T[a, 1] * y) + T[a, 2] * d) + T[a, 3]
                    lo.append(int(np.floor((p - P.trunc) / P.bl)))
                    hi.append(int(np.floor((p + P.trunc) / P.bl)))
                for bx in range(lo[0], hi[0] + 1):
                    for by in range(lo[1], hi[1] + 1):
                        for bz in range(lo[2], hi[2] + 1):
                            want.add((bx, by, bz))
        got = {tuple(b) for b in ot.unpack(keys[(masks[:, k >> 5] >> np.uint32(k & 31)) & 1 == 1])}
        assert got == want and len(want) > 50


def test_fronto_parallel_plane_analytic_tsdf():
    # camera at the origin looking down +z (open3d axes), a plane at z = 1.2, two identical
    # frames: weight 2 and the single-frame tsdf everywhere the plane's band is observed
    H, W = 48, 64
    intr = (50.0, 50.0, 31.5, 23.5)
    P = ot.Params(intr)
    depth = np.full((2, H, W), 1.2, f32)
    color = np.zeros((2, H, W, 3), np.uint8)
    color[..., 0], color[..., 1], color[..., 2] = 10, 200, 77
    c2w = np.tile(np.eye(4, dtype=f32), (2, 1, 1))
    vol = ot.Volume(P)
    vol.integrate(depth, color, c2w, np.linalg.inv(c2w.astype(np.float64)).astype(f32))
    b = np.repeat(ot.unpack(vol.keys), ot.NVOX, 0)
    loc = np.tile(ot._local(), (vol.keys.size, 1))
    cen = (b * 16 + loc + 0.5) * float(P.vl)
    z = cen[:, 2]
    uf, vf = 50.0 * cen[:, 0] / z + 31.5 + 0.5, 50.0 * cen[:, 1] / z + 23.5 + 0.5
    u, v = np.floor(uf), np.floor(vf)
    seen = (z > 0) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    sdf = (1.2 - z) * np.sqrt(((u - 31.5) / 50.0) ** 2 + ((v - 23.5) / 50.0) ** 2 + 1)
    band = seen & (sdf > -0.04)
    assert band.sum() > 10000
    # float32 and float64 may only disagree at the truncation edge or on a pixel-rounding tie
    off = (vol.weight > 0) != band
    tie = (np.abs(uf - np.round(uf)) < 1e-4) | (np.abs(vf - np.round(vf)) < 1e-4)
    assert np.all((np.abs(sdf[off] + 0.04) < 1e-5) | tie[off])
    band &= ~off
    assert np.all(vol.weight[band] == 2)
    t = np.minimum(1.0, sdf[band] / 0.04)
    assert np.abs(vol.tsdf[band] - t).max() < 1e-5
    assert np.all(vol.color[band] == np.array([10, 200, 77], f32))
    # the extracted surface is the plane z = 1.2 (within rounding), normals toward the camera
    verts, faces, cols = vol.extract()
    assert faces.shape[0] > 500
    assert np.abs(verts[:, 2] - 1.2).max() < 1e-5
    n = np.cross(verts[faces[:, 1]] - verts[faces[:, 0]], verts[faces[:, 2]] - verts[faces[:, 0]])
    assert np.all(n[:, 2] < 0)
    assert np.abs(cols * 255 - np.array([10, 200, 77])).max() < 1e-3


def _box_dist(p, box):
    """Distance from points to the surface of an axis-aligned box."""
    lo, hi = box[:, 0], box[:, 1]
    out = np.maximum(np.maximum(lo - p, p - hi), 0)
    outside = np.linalg.norm(out, axis=1)
    inside = np.min(np.minimum(p - lo, hi - p), axis=1)
    return np.where(np.any(out > 0, 1), outside, inside)


def test_synthetic_room_mesh_topology_and_geometry():
    from xrdslam_b200.synthetic import BOXES, ROOM
    cam, poses, depth, color, c2w, w2c = _room(3)
    P = ot.Params(cam)
    vol = ot.Volume(P)
    vol.integrate(depth, color, c2w, w2c)
    verts, faces, cols = vol.extract()
    assert faces.shape[0] > 5000
    # every vertex is referenced
    assert np.array_equal(np.unique(faces), np.arange(verts.shape[0]))
    # every edge bounds at most two faces; interior edges are traversed once each way.  The
    # shared case table (csrc/mc_table.cuh) can put a triangle flat into a cube face whose four
    # edges are crossed; the cube on the other side then emits the same triangle reversed.
    # Such mirror pairs are set aside first, and they must be flat in a lattice plane.
    key = np.sort(faces, 1)
    _, inv, cnt = np.unique(key, axis=0, return_inverse=True, return_counts=True)
    pair = cnt[inv.reshape(-1)] == 2
    assert pair.sum() < 1e-3 * faces.shape[0]
    pv = verts[faces[pair]]
    assert np.all(np.any(np.ptp(pv, axis=1) == 0, axis=1))
    und, directed = edge_use(faces[~pair])
    assert max(und.values()) <= 2
    for (a, b), c in und.items():
        if c == 2:
            assert directed.get((a, b), 0) == 1 and directed.get((b, a), 0) == 1
    # vertices lie on the room walls or the box faces.  The sdf is read at the nearest pixel,
    # so on walls seen at a grazing angle at 160x120 the surface steps by up to about a pixel's
    # depth change: measured median 0.45 voxel, 90th percentile 1.3 voxels, 99.99th 3.3 voxels
    d = np.min(np.stack([np.abs(np.abs(verts - ROOM.mean(1)) - (ROOM[:, 1] - ROOM[:, 0]) / 2).min(1)]
                        + [_box_dist(verts.astype(np.float64), b) for b in BOXES]), 0)
    vl = float(P.vl)
    assert np.median(d) < 0.5 * vl and np.quantile(d, 0.9) < 1.5 * vl
    assert np.quantile(d, 0.999) < 0.04 and d.max() < 0.06
    # normals point to the free side, towards the cameras (area-weighted; the steps above and
    # the room's concave corners hold the faces that do not: measured 7.7 %)
    eye = np.mean([p[:3, 3] for p in poses], 0)
    a, b, c = (verts[faces[:, i]].astype(np.float64) for i in range(3))
    n = np.cross(b - a, c - a)
    area = np.linalg.norm(n, axis=1)
    toward = np.einsum('ij,ij->i', n, eye - (a + b + c) / 3) > 0
    assert area[toward].sum() > 0.9 * area.sum()
    assert cols.min() >= 0 and cols.max() <= 1


def test_components_match_scipy():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    cam, _, depth, color, c2w, w2c = _room(2)
    vol = ot.Volume(ot.Params(cam))
    vol.integrate(depth, color, c2w, w2c)
    verts, faces, _ = vol.extract()
    rng = np.random.default_rng(0)
    for f, n in ((faces, verts.shape[0]),
                 (rng.integers(0, 3000, (1500, 3)), 3000)):   # many small components
        lab = ot.components(f, n)
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n))
        nc, sl = connected_components(g, directed=False)
        assert len(np.unique(lab)) == nc
        # same partition, labelled by the smallest member
        mins = np.full(nc, n)
        np.minimum.at(mins, sl, np.arange(n))
        assert np.array_equal(lab, mins[sl])


def _strip(n_verts, x0):
    """A triangle strip with n_verts vertices (one component) at x offset x0."""
    k = n_verts // 2
    top = np.stack([np.arange(k) + x0, np.zeros(k), np.zeros(k)], 1)
    bot = np.stack([np.arange(n_verts - k) + x0, np.ones(n_verts - k), np.zeros(n_verts - k)], 1)
    v = np.concatenate([top, bot]).astype(f32)
    f = [[i, k + i, i + 1] for i in range(k - 1)] + [[i + 1, k + i, k + i + 1]
                                                     for i in range(min(k - 1, n_verts - k - 1))]
    return v, np.array(f)


def test_clean_mesh_keeps_components_of_at_least_100_vertices():
    v99, f99 = _strip(99, 0.0)
    v100, f100 = _strip(100, 1000.0)
    v = np.concatenate([v99, v100])
    f = np.concatenate([f99, f100 + 99])
    # a duplicate face, a face that collapses once two bit-identical vertices are welded
    v = np.concatenate([v, v100[:1]])
    f = np.concatenate([f, f100[:1] + 99, [[99, 100, v.shape[0] - 1]]])
    c = np.random.default_rng(0).random(v.shape, dtype=f32)
    cv, cf, cc = ot.clean_mesh(v, f, c)
    assert cv.shape[0] == 100 and np.array_equal(cv, v100)
    assert cf.shape[0] == f100.shape[0] and np.array_equal(cf, f100)
    assert np.array_equal(cc, c[99:199])
