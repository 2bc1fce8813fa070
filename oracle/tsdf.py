"""numpy float32 restatement of the block-sparse TSDF fusion, its coloured marching cubes and
clean_mesh (csrc/tsdf.cu, xrdslam_b200/tsdf.py; semantics in include/xrdslam_b200.h).

ORACLE / TEST INFRASTRUCTURE -- never imported by xrdslam_b200/.

Every float32 operation is written in the kernels' order, so the results match bit for bit:
  allocation   x = ((u - cx) * d) / fx,  p = ((T0*x + T1*y) + T2*z) + T3,
               blocks floor((p -/+ sdf_trunc) / bl) per axis
  integration  centre = b*bl + (i + 0.5)*vl; (x, y, z) = w2c * centre; u = floor(fx*x/z + cx
               + 0.5); sdf = (d - z) * sqrt((qa*qa + qb*qb) + 1); t = min(1, sdf / trunc);
               running averages (v*w + new) / (w + 1)
  extraction   t = (0 - v0) / (v1 - v0); position ((c*vl + vl*0.5)*1) + b*bl; colour
               (c0 + t*(c1 - c0)) / 255
"""
from __future__ import annotations

import numpy as np

from oracle.mc_table import EDGE_AXIS, EDGE_OFF
from oracle.marching_cubes import _POP, NTRI, TRI

f32 = np.float32
RES = 16
NVOX = RES ** 3
BIAS = 1 << 20
_EAX = np.asarray(EDGE_AXIS, np.int64)
_EOFF = np.asarray(EDGE_OFF, np.int64)
# EUSE[case, e]: edge e is referenced by a triangle of the case
EUSE = np.zeros((256, 12), bool)
for _c in range(256):
    for _e in TRI[_c][:NTRI[_c]].reshape(-1):
        EUSE[_c, _e] = True


class Params:
    def __init__(self, camera_or_intrinsic, voxel_length=4.0 / 512.0, sdf_trunc=0.04,
                 depth_trunc=1000.0, stride=4):
        c = camera_or_intrinsic
        fx, fy, cx, cy = (c.fx, c.fy, c.cx, c.cy) if hasattr(c, 'fx') else c
        self.fx, self.fy, self.cx, self.cy = f32(fx), f32(fy), f32(cx), f32(cy)
        self.vl, self.trunc, self.dtrunc = f32(voxel_length), f32(sdf_trunc), f32(depth_trunc)
        self.bl = self.vl * f32(RES)
        self.stride = int(stride)


def pack(b):
    b = np.asarray(b, np.int64) + BIAS
    return (b[..., 0] << 42) | (b[..., 1] << 21) | b[..., 2]


def unpack(k):
    k = np.asarray(k, np.int64)
    m = (1 << 21) - 1
    return np.stack([(k >> 42) & m, (k >> 21) & m, k & m], -1) - BIAS


def xform(T, r, x, y, z):
    T = np.asarray(T, f32)
    return ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]


def depth_ok(d, P):
    return (d > 0) & ~(d > P.dtrunc)


def frame_blocks(depth, c2w, P):
    """Keys of the blocks one frame touches (not unique) -> int64 [m]."""
    H, W = depth.shape
    v, u = np.meshgrid(np.arange(0, H, P.stride), np.arange(0, W, P.stride), indexing='ij')
    d = depth[v, u].astype(f32)
    ok = depth_ok(d, P)
    u, v, d = u[ok].astype(f32), v[ok].astype(f32), d[ok]
    x = ((u - P.cx) * d) / P.fx
    y = ((v - P.cy) * d) / P.fy
    p = np.stack([xform(c2w, a, x, y, d) for a in range(3)], -1)
    with np.errstate(invalid='ignore'):
        lo = np.floor((p - P.trunc) / P.bl)
        hi = np.floor((p + P.trunc) / P.bl)
        ok = np.all((lo >= f32(-BIAS)) & (hi < f32(BIAS - 1)), 1)
    lo, hi = lo[ok].astype(np.int64), hi[ok].astype(np.int64)
    n = np.minimum(hi - lo, 1) + 1
    out = []
    for dx in range(2):
        for dy in range(2):
            for dz in range(2):
                m = (dx < n[:, 0]) & (dy < n[:, 1]) & (dz < n[:, 2])
                out.append(pack(lo[m] + np.array([dx, dy, dz])))
    return np.concatenate(out)


def allocate(depth, c2w, P):
    """depth f32 [K,H,W], c2w f32 [K,>=3,4] -> keys int64 [n] sorted, masks uint32 [n, words]."""
    K = depth.shape[0]
    per = [np.unique(frame_blocks(depth[k], c2w[k], P)) for k in range(K)]
    keys = np.unique(np.concatenate(per)) if per else np.zeros(0, np.int64)
    masks = np.zeros((keys.size, (K + 31) // 32), np.uint32)
    for k, kk in enumerate(per):
        r = np.searchsorted(keys, kk)
        masks[r, k >> 5] |= np.uint32(1 << (k & 31))
    return keys, masks


def _local():
    v = np.arange(NVOX)
    return np.stack([v >> 8, (v >> 4) & 15, v & 15], -1)


class Volume:
    """The restated volume: keys int64 [n], tsdf / weight f32 [n*4096], color f32 [n*4096,3]."""

    def __init__(self, P):
        self.P = P
        self.keys = np.zeros(0, np.int64)
        self.tsdf = np.zeros(0, f32)
        self.weight = np.zeros(0, f32)
        self.color = np.zeros((0, 3), f32)

    def integrate(self, depth, color, c2w, w2c):
        P = self.P
        depth = np.asarray(depth, f32)
        color = np.asarray(color, np.uint8)
        keys, masks = allocate(depth, c2w, P)
        if keys.size == 0:
            return keys, masks
        union = np.union1d(self.keys, keys)
        if union.size != self.keys.size:
            n = union.size
            t, w, c = np.zeros((n, NVOX), f32), np.zeros((n, NVOX), f32), np.zeros((n, NVOX, 3), f32)
            old = np.searchsorted(union, self.keys)
            t[old] = self.tsdf.reshape(-1, NVOX)
            w[old] = self.weight.reshape(-1, NVOX)
            c[old] = self.color.reshape(-1, NVOX, 3)
            self.keys, self.tsdf, self.weight, self.color = (union, t.reshape(-1), w.reshape(-1),
                                                             c.reshape(-1, 3))
        rows = np.searchsorted(self.keys, keys)
        loc = _local().astype(f32) + f32(0.5)
        K, H, W = depth.shape
        for k in range(K):
            blocks = rows[(masks[:, k >> 5] >> np.uint32(k & 31)) & np.uint32(1) == 1]
            if blocks.size == 0:
                continue
            bk = unpack(self.keys[blocks]).astype(f32)                    # [m,3]
            cen = bk[:, None, :] * P.bl + loc[None] * P.vl                 # [m,4096,3]
            g = (blocks[:, None] * NVOX + np.arange(NVOX)[None]).reshape(-1)
            cen = cen.reshape(-1, 3)
            T = np.asarray(w2c[k], f32)
            z = xform(T, 2, cen[:, 0], cen[:, 1], cen[:, 2])
            x = xform(T, 0, cen[:, 0], cen[:, 1], cen[:, 2])
            y = xform(T, 1, cen[:, 0], cen[:, 1], cen[:, 2])
            with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
                fu = np.floor(((P.fx * x) / z + P.cx) + f32(0.5))
                fv = np.floor(((P.fy * y) / z + P.cy) + f32(0.5))
            ok = (z > 0) & (fu >= 0) & (fu < f32(W)) & (fv >= 0) & (fv < f32(H))
            g, z, fu, fv = g[ok], z[ok], fu[ok], fv[ok]
            ui, vi = fu.astype(np.int64), fv.astype(np.int64)
            d = depth[k, vi, ui]
            ok = depth_ok(d, P)
            g, z, fu, fv, ui, vi, d = g[ok], z[ok], fu[ok], fv[ok], ui[ok], vi[ok], d[ok]
            qa = (fu - P.cx) / P.fx
            qb = (fv - P.cy) / P.fy
            sdf = (d - z) * np.sqrt((qa * qa + qb * qb) + f32(1))
            ok = ~(sdf <= -P.trunc)
            g, sdf, ui, vi = g[ok], sdf[ok], ui[ok], vi[ok]
            t = np.minimum(f32(1), sdf / P.trunc)
            w = self.weight[g]
            w1 = w + f32(1)
            self.tsdf[g] = (self.tsdf[g] * w + t) / w1
            ck = color[k, vi, ui].astype(f32)
            self.color[g] = (self.color[g] * w[:, None] + ck) / w1[:, None]
            self.weight[g] = w1
        return keys, masks

    def extract(self, chunk=1024):
        return extract(self.keys, self.tsdf, self.weight, self.color, self.P.vl, chunk)


def neighbours(keys):
    """nbr int64 [n, 8]: column c = block at offset (c>>2&1, c>>1&1, c&1), -1 if missing."""
    b = unpack(keys)
    nbr = np.empty((keys.size, 8), np.int64)
    for c in range(8):
        q = b + np.array([(c >> 2) & 1, (c >> 1) & 1, c & 1])
        inr = np.all(q < BIAS, 1)
        qk = pack(np.where(inr[:, None], q, 0))
        r = np.searchsorted(keys, qk)
        rc = np.minimum(r, keys.size - 1)
        nbr[:, c] = np.where(inr & (r < keys.size) & (keys[rc] == qk), rc, -1)
    return nbr


def voxel_at(nbr, b, i, j, k):
    c = ((i >> 4) << 2) | ((j >> 4) << 1) | (k >> 4)
    nb = nbr[b, c]
    q = nb * NVOX + ((i & 15) << 8) + ((j & 15) << 4) + (k & 15)
    return np.where(nb >= 0, q, -1)


def classify(keys, tsdf, weight, nbr, chunk=1024):
    """-> case uint8 [n*4096], ntri int64 [n*4096] (0 for unused cubes)."""
    n = keys.size * NVOX
    cases = np.zeros(n, np.uint8)
    ntri = np.zeros(n, np.int64)
    loc = _local()
    for b0 in range(0, keys.size, chunk):
        b1 = min(keys.size, b0 + chunk)
        b = np.repeat(np.arange(b0, b1), NVOX)
        l = np.tile(loc, (b1 - b0, 1))
        cs = np.zeros(b.size, np.int64)
        used = np.ones(b.size, bool)
        for c in range(8):
            q = voxel_at(nbr, b, l[:, 0] + ((c >> 2) & 1), l[:, 1] + ((c >> 1) & 1),
                         l[:, 2] + (c & 1))
            qq = np.maximum(q, 0)
            used &= (q >= 0) & (weight[qq] > 0)
            cs |= (tsdf[qq] < 0).astype(np.int64) << c
        sl = slice(b0 * NVOX, b1 * NVOX)
        cases[sl] = cs
        ntri[sl] = np.where(used, NTRI[cs], 0)
    return cases, ntri


def extract(keys, tsdf, weight, color, vl, chunk=1024):
    """-> verts f32 [V,3], faces int32 [F,3], colors f32 [V,3]."""
    vl = f32(vl)
    if keys.size == 0:
        return np.zeros((0, 3), f32), np.zeros((0, 3), np.int32), np.zeros((0, 3), f32)
    nbr = neighbours(keys)
    cases, ntri = classify(keys, tsdf, weight, nbr, chunk)
    n = keys.size * NVOX
    cubes = np.nonzero(ntri)[0]
    cb, cv = cubes >> 12, cubes & (NVOX - 1)
    ci, cj, ck = cv >> 8, (cv >> 4) & 15, cv & 15
    own = [np.zeros(n, bool) for _ in range(3)]
    for e in range(12):
        m = EUSE[cases[cubes], e]
        q = voxel_at(nbr, cb[m], ci[m] + _EOFF[e, 0], cj[m] + _EOFF[e, 1], ck[m] + _EOFF[e, 2])
        own[_EAX[e]][q] = True
    flags = own[0].astype(np.int64) | (own[1].astype(np.int64) << 1) | (own[2].astype(np.int64) << 2)
    vcnt = own[0].astype(np.int64) + own[1] + own[2]
    vbase = np.concatenate([[0], np.cumsum(vcnt)[:-1]])
    V = int(vcnt.sum())
    verts = np.empty((V, 3), f32)
    cols = np.empty((V, 3), f32)
    bl = vl * f32(RES)
    half = vl * f32(0.5)
    for a in range(3):
        p = np.nonzero(own[a])[0]
        ids = vbase[p] + sum(own[x][p].astype(np.int64) for x in range(a))
        b, v = p >> 12, p & (NVOX - 1)
        idx = np.stack([v >> 8, (v >> 4) & 15, v & 15], 1)
        q = voxel_at(nbr, b, *(idx[:, x] + (x == a) for x in range(3)))
        v0, v1 = tsdf[p], tsdf[q]
        t = (f32(0) - v0) / (v1 - v0)
        c = idx.astype(f32)
        c[:, a] = c[:, a] + t
        o = unpack(keys[b]).astype(f32) * bl
        verts[ids] = ((c * vl + half) * f32(1)) + o
        k0, k1 = color[p], color[q]
        cols[ids] = (k0 + t[:, None] * (k1 - k0)) / f32(255)
    nt = ntri[cubes]
    pc = np.repeat(np.arange(cubes.size), nt)
    start = np.concatenate([[0], np.cumsum(nt)[:-1]])
    tt = np.arange(pc.size) - np.repeat(start, nt)
    e = TRI[cases[cubes][pc], tt]                          # [F,3]
    faces = np.empty(e.shape, np.int64)
    for m in range(3):
        em = e[:, m]
        q = voxel_at(nbr, cb[pc], ci[pc] + _EOFF[em, 0], cj[pc] + _EOFF[em, 1], ck[pc] + _EOFF[em, 2])
        ax = _EAX[em]
        faces[:, m] = vbase[q] + _POP[flags[q] & ((1 << ax) - 1)]
    return verts, faces.astype(np.int32).reshape(-1, 3), cols


# ---- clean_mesh --------------------------------------------------------------------------------
def components(faces, n_verts):
    """labels int64 [n_verts]: the smallest vertex id connected through face edges."""
    lab = np.arange(n_verts, dtype=np.int64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    while True:
        while True:                                  # pointer jumping to the roots
            nl = lab[lab]
            if np.array_equal(nl, lab):
                break
            lab = nl
        ra, rb = lab[a], lab[b]
        if np.array_equal(ra, rb):
            return lab
        m = np.minimum(ra, rb)
        np.minimum.at(lab, ra, m)                     # hook every root below the smaller one
        np.minimum.at(lab, rb, m)


def clean_mesh(verts, faces, colors, min_len=100):
    """-> verts f32, faces int32, colors f32 (semantics of xrdslam_b200.tsdf.clean_mesh_arrays)."""
    verts = np.ascontiguousarray(verts, f32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    if verts.shape[0] == 0 or faces.shape[0] == 0:
        return verts[:0], faces[:0].astype(np.int32), np.asarray(colors, f32)[:0]
    _, first, inv = np.unique(verts.view(np.int32), axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(first, kind='stable')
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    src = first[order]
    wv, wc = verts[src], np.asarray(colors, f32)[src]
    wf = rank[inv][faces]
    n = wv.shape[0]
    lab = components(wf, n)
    ref = np.zeros(n, bool)
    ref[wf.reshape(-1)] = True
    size = np.bincount(lab[ref], minlength=n)
    keep = ref & (size[lab] >= min_len)
    vid = np.nonzero(keep)[0]
    vid = vid[np.argsort(lab[vid], kind='stable')]
    new = -np.ones(n, np.int64)
    new[vid] = np.arange(vid.size)
    fid = np.nonzero(keep[wf[:, 0]])[0]
    fid = fid[np.argsort(lab[wf[fid, 0]], kind='stable')]
    nf = new[wf[fid]]
    nf = nf[(nf[:, 0] != nf[:, 1]) & (nf[:, 1] != nf[:, 2]) & (nf[:, 0] != nf[:, 2])]
    if nf.shape[0]:
        _, ff = np.unique(np.sort(nf, 1), axis=0, return_index=True)
        nf = nf[np.sort(ff)]
    return wv[vid], nf.astype(np.int32), wc[vid]


def colors_to_u8(c):
    return (np.clip(c, 0, 1) * f32(255)).astype(np.uint8)


def o3d_poses(c2w_list):
    c2w = np.stack([np.asarray(p, f32).reshape(4, 4) for p in c2w_list]).copy()
    c2w[:, :3, 1] *= f32(-1)
    c2w[:, :3, 2] *= f32(-1)
    return c2w, np.linalg.inv(c2w.astype(np.float64)).astype(f32)
