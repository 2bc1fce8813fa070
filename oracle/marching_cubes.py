"""numpy float32 restatement of the CUDA marching cubes (csrc/mesh.cu).

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Same table (oracle/mc_table.py), same vertex and face order, same float32 operations:
  t      = (level - v0) / (v1 - v0)                    on the crossed lattice edge v0 -> v1
  p[a]   = index[a] (+ t on the edge's axis)
  world  = ((p * spacing + shift) * scale) + origin[b]  rounded after every operation
Vertices are ordered by (volume, flat lattice index of the edge's lower endpoint, axis x/y/z),
faces by (volume, cube = flat index of its lower lattice point, triangle within the case).
"""
from __future__ import annotations

import numpy as np

from oracle.mc_table import EDGE_AXIS, EDGE_OFF, build

f32 = np.float32
_TABLES = build()
MAX_TRI = max(len(t) for t in _TABLES)
NTRI = np.array([len(t) for t in _TABLES], np.int64)
TRI = -np.ones((256, MAX_TRI, 3), np.int64)
for _c, _t in enumerate(_TABLES):
    if _t:
        TRI[_c, :len(_t)] = np.array(_t)
_POP = np.array([bin(i).count('1') for i in range(8)], np.int64)


def marching_cubes(values, level, spacing, shift=(0, 0, 0), scale=(1, 1, 1), origin=None):
    """values float32 [B, nx, ny, nz] (x slowest) -> verts f32 [V,3], faces i32 [F,3]."""
    v = np.ascontiguousarray(values, dtype=f32)
    B, nx, ny, nz = v.shape
    lev = f32(level)
    neg = v < lev
    strides = np.array([ny * nz, nz, 1], np.int64)
    # owned crossed edges of every lattice point: bit a for the edge along axis a
    flags = np.zeros(v.shape, np.int64)
    flags[:, :-1] |= (neg[:, :-1] != neg[:, 1:]).astype(np.int64)
    flags[:, :, :-1] |= (neg[:, :, :-1] != neg[:, :, 1:]).astype(np.int64) << 1
    flags[:, :, :, :-1] |= (neg[:, :, :, :-1] != neg[:, :, :, 1:]).astype(np.int64) << 2
    flat_flags = flags.reshape(-1)
    vcnt = _POP[flat_flags]
    vbase = np.concatenate([[0], np.cumsum(vcnt)[:-1]]).astype(np.int64)
    V = int(vcnt.sum())
    vf = v.reshape(-1)
    sp, sh, sc = (np.asarray(a, f32).reshape(3) for a in (spacing, shift, scale))
    org = np.zeros((B, 3), f32) if origin is None else np.asarray(origin, f32).reshape(B, 3)

    verts = np.empty((V, 3), f32)
    for a in range(3):
        p = np.nonzero(flat_flags & (1 << a))[0]
        ids = vbase[p] + _POP[flat_flags[p] & ((1 << a) - 1)]
        b, rem = np.divmod(p, nx * ny * nz)
        idx = np.stack([rem // (ny * nz), (rem // nz) % ny, rem % nz], 1).astype(f32)
        v0, v1 = vf[p], vf[p + strides[a]]
        t = (lev - v0) / (v1 - v0)
        idx[:, a] = idx[:, a] + t
        w = ((idx * sp) + sh) * sc
        verts[ids] = w + org[b]

    # cubes: lower lattice point with a full cube above it
    c = np.zeros((B, nx - 1, ny - 1, nz - 1), np.int64)
    for k in range(8):
        dx, dy, dz = (k >> 2) & 1, (k >> 1) & 1, k & 1
        c |= neg[:, dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.int64) << k
    cases = np.zeros(v.shape, np.int64)
    cases[:, :-1, :-1, :-1] = c
    cases = cases.reshape(-1)
    nt = NTRI[cases]
    p = np.repeat(np.arange(cases.size, dtype=np.int64), nt)
    start = np.concatenate([[0], np.cumsum(nt)[:-1]])
    t = np.arange(p.size) - np.repeat(start, nt)
    e = TRI[cases[p], t]                                    # [F,3] edge ids
    axis = np.asarray(EDGE_AXIS, np.int64)[e]
    q = p[:, None] + np.asarray(EDGE_OFF, np.int64)[e] @ strides
    faces = vbase[q] + _POP[flat_flags[q] & ((1 << axis) - 1)]
    return verts, faces.astype(np.int32).reshape(-1, 3)


# ---- analytic checks used by the tests ----------------------------------------------------
def edge_use(faces):
    """(undirected edge -> face count, directed edge -> count)."""
    from collections import Counter
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    directed = Counter(map(tuple, d.tolist()))
    undirected = Counter(map(tuple, np.sort(d, 1).tolist()))
    return undirected, directed


def euler_characteristic(verts, faces):
    und, _ = edge_use(faces)
    used = np.unique(faces)
    return int(used.size) - len(und) + int(faces.shape[0])


def signed_volume(verts, faces):
    a, b, c = (verts[faces[:, i]].astype(np.float64) for i in range(3))
    return float(np.einsum('ij,ij->i', a, np.cross(b, c)).sum() / 6.0)
